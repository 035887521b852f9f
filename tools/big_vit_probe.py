"""ViT-H-14, ViT-g-14 and ViT-bigG-14 image forwards on one GPU: the engine at b256 (device-resident uint8 at the model's
size) against torch running the same weights (the oracle's arithmetic, attention through scaled_dot_product_attention)
under bf16 autocast, the two alternated in one process (`--warmup` and `--steps` calls each); torch runs b64 where b256
does not fit.  Also prints the card and its power limit, each kernel class's share of the engine's forward (a
torch.profiler run of its own), debug_attention_time at the padded head dims against head dim 64, and the FLOPs the
zero-padded heads add, computed from the shapes.

    python tools/big_vit_probe.py [--steps 10] [--warmup 2] [--models h14,h14_378,g14,bigg] [--out FILE]

The results are printed; --out also writes them to FILE as JSON."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from marqo_b200 import model_registry as R  # noqa: E402
from marqo_b200.engine import Encoder, debug_attention_time  # noqa: E402
from marqo_b200.weights import random_clip_weights  # noqa: E402

B = 256
NAMES = {"h14": "open_clip/ViT-H-14/laion2b_s32b_b79k", "h14_378": "open_clip/ViT-H-14-378-quickgelu/dfn5b",
         "g14": "open_clip/ViT-g-14/laion2b_s12b_b42k", "bigg": "open_clip/ViT-bigG-14/laion2b_s39b_b160k"}
MEAN = torch.tensor(R.OPENAI_MEAN).view(1, 3, 1, 1)
STD = torch.tensor(R.OPENAI_STD).view(1, 3, 1, 1)


def kernel_head_dim(hd):
    return hd if hd <= 64 else 96 if hd <= 96 else 128


def padding_flops(v):
    """Per layer and image: (GEMM FLOPs unpadded, padded), (attention FLOPs unpadded, padded)."""
    w, H, mlp = v["width"], v["heads"], v["mlp"]
    S = (v["image_size"] // v["patch"]) ** 2 + 1
    hd = w // H
    aw = H * kernel_head_dim(hd)
    gemm = lambda a: 2 * S * (3 * a * w + a * w + 2 * w * mlp)   # noqa: E731  QKV, out-proj, fc1, fc2
    attn = lambda d: 2 * 2 * S * S * H * d                       # noqa: E731  QK^T and P V
    return (gemm(w), gemm(aw)), (attn(hd), attn(kernel_head_dim(hd)))


def torch_vision(sd, a, x):
    """open_clip's VisionTransformer forward (the oracle's), attention through scaled_dot_product_attention."""
    v = a["vision"]
    w, H = v["width"], v["heads"]
    x = F.conv2d(x, sd["visual.conv1.weight"], None, stride=v["patch"])
    n = x.shape[0]
    x = x.reshape(n, w, -1).permute(0, 2, 1)
    x = torch.cat([sd["visual.class_embedding"].to(x.dtype).expand(n, 1, w), x], 1) + sd["visual.positional_embedding"]
    x = F.layer_norm(x, (w,), sd["visual.ln_pre.weight"], sd["visual.ln_pre.bias"], 1e-5)
    for i in range(v["layers"]):
        p = f"visual.transformer.resblocks.{i}."
        h = F.layer_norm(x, (w,), sd[p + "ln_1.weight"], sd[p + "ln_1.bias"], 1e-5)
        q, k, vv = F.linear(h, sd[p + "attn.in_proj_weight"], sd[p + "attn.in_proj_bias"]).split(w, -1)
        q, k, vv = (t.view(n, -1, H, w // H).transpose(1, 2) for t in (q, k, vv))
        o = F.scaled_dot_product_attention(q, k, vv).transpose(1, 2).reshape(n, -1, w)
        x = x + F.linear(o, sd[p + "attn.out_proj.weight"], sd[p + "attn.out_proj.bias"])
        h = F.layer_norm(x, (w,), sd[p + "ln_2.weight"], sd[p + "ln_2.bias"], 1e-5)
        h = F.linear(h, sd[p + "mlp.c_fc.weight"], sd[p + "mlp.c_fc.bias"])
        h = h * torch.sigmoid(1.702 * h) if a["act"] == "quickgelu" else F.gelu(h)
        x = x + F.linear(h, sd[p + "mlp.c_proj.weight"], sd[p + "mlp.c_proj.bias"])
    pooled = F.layer_norm(x[:, 0], (w,), sd["visual.ln_post.weight"], sd["visual.ln_post.bias"], 1e-5)
    out = (pooled @ sd["visual.proj"]).float()
    return out / out.norm(dim=-1, keepdim=True)


def events_ms(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e)


def kernel_class(name):
    for key, cls in (("gemm", "gemm"), ("attention", "attention"), ("layernorm", "layernorm")):
        if key in name:
            return cls
    return "other"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--models", default="h14,h14_378,g14,bigg")
    ap.add_argument("--out")
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    res = {"card": q, "batch": B, "models": {}, "attention": {}}
    print("card:", q, flush=True)
    for S, H, hd in ((257, 16, 64), (257, 16, 96), (730, 16, 96), (257, 16, 128), (730, 16, 64)):
        ms = debug_attention_time(B, S, H * hd, H, 0, iters=50)
        res["attention"][f"S{S}_H{H}_hd{hd}"] = {"ms": ms, "TFLOP_s": 4 * B * S * S * H * hd / ms / 1e9}
        print(f"attention b{B} S={S} H={H} hd={hd}: {ms:.3f} ms", flush=True)
    for key in args.models.split(","):
        arch = R.get_model_properties(NAMES[key])["arch"]
        arch["text"] = None
        v, E = arch["vision"], arch["embed_dim"]
        S = v["image_size"]
        (g0, g1), (a0, a1) = padding_flops(v)
        t0 = time.time()
        sd = random_clip_weights(arch, seed=1)
        enc = Encoder("clip", arch, sd, max_batch=B)
        enc.set_stream(torch.cuda.current_stream().cuda_stream)   # the events below time the engine's own launches
        print(f"{key}: weights + finalize {time.time() - t0:.1f} s", flush=True)
        tsd = {k: torch.as_tensor(val).cuda() for k, val in sd.items()}
        del sd
        img = torch.randint(0, 256, (B, S, S, 3), dtype=torch.uint8, device="cuda")
        out = torch.empty((B, E), device="cuda")

        def engine():
            enc.encode_images_u8_device(img.data_ptr(), B, S, S, out.data_ptr(), sync=False)

        tb = B

        def reference():
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                for i in range(0, B, tb):
                    x = (img[i:i + tb].permute(0, 3, 1, 2).float() / 255 - MEAN.cuda()) / STD.cuda()
                    torch_vision(tsd, arch, x)

        try:
            reference()
        except torch.OutOfMemoryError:
            tb = 64
            torch.cuda.empty_cache()
        for _ in range(args.warmup):
            engine()
            reference()
        torch.cuda.synchronize()
        te, tr = [], []
        for _ in range(args.steps):
            te.append(events_ms(engine))
            tr.append(events_ms(reference))
        with torch.no_grad():
            x = (img[:4].permute(0, 3, 1, 2).float() / 255 - MEAN.cuda()) / STD.cuda()
            old = torch.backends.cuda.matmul.allow_tf32
            torch.backends.cuda.matmul.allow_tf32 = False
            ref = torch_vision(tsd, arch, x)
            torch.backends.cuda.matmul.allow_tf32 = old
        cos = float(F.cosine_similarity(out[:4].double(), ref.double(), dim=-1).min())
        fwd_ms = float(np.median(te))
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            engine()
            torch.cuda.synchronize()
        cls_us = {}
        for ev in prof.key_averages():
            t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            if ev.key.startswith(("Memcpy", "Memset")) or t <= 0:
                continue
            c = kernel_class(ev.key)
            cls_us[c] = cls_us.get(c, 0.0) + t
        total = sum(cls_us.values())
        layer_flops = (g1 + a1) * B * v["layers"]
        r = {"engine_ms": fwd_ms, "torch_bf16_sdpa_ms": float(np.median(tr)), "torch_batch": tb,
             "engine_img_s": B / fwd_ms * 1e3, "min_cosine_vs_torch_fp32": cos,
             "layers_TFLOP_s": layer_flops / fwd_ms / 1e9,
             "kernel_share": {c: us / total for c, us in sorted(cls_us.items())},
             "padding_extra_flops": {"gemm": g1 / g0 - 1, "attention": a1 / a0 - 1}}
        res["models"][key] = r
        print(key, json.dumps(r, indent=1), flush=True)
        enc.close()
        del tsd
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
