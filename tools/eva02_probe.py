"""EVA02-B-16, EVA02-L-14 and EVA02-L-14-336 image forwards on one GPU: the engine at b256 (device-resident uint8 at
the model's size, seeded weights) against torch running the same weights (the tests' fp32 restatement, attention
through scaled_dot_product_attention) under bf16 autocast, the two alternated in one process (`--warmup` and `--steps`
calls each, medians reported); torch runs b64 where b256 does not fit.  Also prints the card's name and power limit,
read in the same process, and each kernel class's share of the engine's forward (GEMM, attention, LayerNorm, rope,
SwiGLU; a torch.profiler run of its own).

    python tools/eva02_probe.py [--steps 10] [--warmup 2] [--models b16,l14,l14_336] [--out FILE]

The results are printed; --out also writes them to FILE as JSON."""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from marqo_b200 import model_registry as R  # noqa: E402
from marqo_b200.engine import Encoder  # noqa: E402
from marqo_b200.weights import random_eva02_weights  # noqa: E402
import _eva02_oracle as V  # noqa: E402

B = 256
NAMES = {"b16": V.B16, "l14": V.L14, "l14_336": V.L14_336}
MEAN = torch.tensor(R.OPENAI_MEAN).view(1, 3, 1, 1)
STD = torch.tensor(R.OPENAI_STD).view(1, 3, 1, 1)


def torch_vision(sd, a, x, sin, cos):
    """The tests' EVA02 restatement (tests/_eva02_oracle.py) with the attention through scaled_dot_product_attention."""
    ev = a["eva"]
    t, W, P, H, eps = "visual.trunk.", ev["width"], ev["patch"], ev["heads"], ev["ln_eps"]
    x = F.conv2d(x, sd[t + "patch_embed.proj.weight"], sd[t + "patch_embed.proj.bias"], stride=P)
    n = x.shape[0]
    x = x.reshape(n, W, -1).permute(0, 2, 1)
    x = torch.cat([sd[t + "cls_token"].to(x.dtype).expand(n, 1, W), x], 1) + sd[t + "pos_embed"]
    for i in range(ev["layers"]):
        p = f"{t}blocks.{i}."
        h = F.layer_norm(x, (W,), sd[p + "norm1.weight"], sd[p + "norm1.bias"], eps)
        q = F.linear(h, sd[p + "attn.q_proj.weight"], sd[p + "attn.q_proj.bias"])
        k = F.linear(h, sd[p + "attn.k_proj.weight"])
        v = F.linear(h, sd[p + "attn.v_proj.weight"], sd[p + "attn.v_proj.bias"])
        q, k, v = (z.view(n, -1, H, 64).transpose(1, 2) for z in (q, k, v))
        q = torch.cat([q[:, :, :1], V.rotate(q[:, :, 1:], sin, cos).to(q.dtype)], 2)
        k = torch.cat([k[:, :, :1], V.rotate(k[:, :, 1:], sin, cos).to(k.dtype)], 2)
        o = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(n, -1, W)
        o = F.layer_norm(o, (W,), sd[p + "attn.norm.weight"], sd[p + "attn.norm.bias"], eps)
        x = x + F.linear(o, sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"])
        h = F.layer_norm(x, (W,), sd[p + "norm2.weight"], sd[p + "norm2.bias"], eps)
        u = F.silu(F.linear(h, sd[p + "mlp.fc1_g.weight"], sd[p + "mlp.fc1_g.bias"])) * F.linear(
            h, sd[p + "mlp.fc1_x.weight"], sd[p + "mlp.fc1_x.bias"])
        u = F.layer_norm(u, (u.shape[-1],), sd[p + "mlp.norm.weight"], sd[p + "mlp.norm.bias"], eps)
        x = x + F.linear(u, sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"])
    x = F.layer_norm(x[:, 0], (W,), sd[t + "norm.weight"], sd[t + "norm.bias"], eps)
    out = F.linear(x, sd[t + "head.weight"], sd[t + "head.bias"]).float()
    return out / out.norm(dim=-1, keepdim=True)


def events_ms(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e)


def kernel_class(name):
    for key, cls in (("gemm", "gemm"), ("attention", "attention"), ("layernorm", "layernorm"), ("rope", "rope"),
                     ("swiglu", "swiglu")):
        if key in name:
            return cls
    return "other"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--models", default="b16,l14,l14_336")
    ap.add_argument("--out")
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    res = {"card": q, "batch": B, "models": {}}
    print("card:", q, flush=True)
    for key in args.models.split(","):
        arch = R.get_model_properties(NAMES[key])["arch"]
        arch["layers"] = 0   # image tower only
        ev, E = arch["eva"], arch["embed_dim"]
        S = ev["image_size"]
        G = S // ev["patch"]
        t0 = time.time()
        sd = random_eva02_weights(arch, seed=1)
        enc = Encoder("clip_eva", arch, sd, max_batch=B)
        enc.set_stream(torch.cuda.current_stream().cuda_stream)   # the events below time the engine's own launches
        print(f"{key}: weights + finalize {time.time() - t0:.1f} s", flush=True)
        tsd = {k: torch.as_tensor(val).cuda() for k, val in sd.items()}
        del sd
        sin, cos = (r.cuda() for r in V.rope_sin_cos(G, ev["rope_ref_grid"]))
        img = torch.randint(0, 256, (B, S, S, 3), dtype=torch.uint8, device="cuda")
        out = torch.empty((B, E), device="cuda")

        def engine():
            enc.encode_images_u8_device(img.data_ptr(), B, S, S, out.data_ptr(), sync=False)

        tb = B

        def reference():
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                for i in range(0, B, tb):
                    x = (img[i:i + tb].permute(0, 3, 1, 2).float() / 255 - MEAN.cuda()) / STD.cuda()
                    torch_vision(tsd, arch, x, sin, cos)

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
            ref = V.encode_image(tsd, arch, x)
            torch.backends.cuda.matmul.allow_tf32 = old
        cos_min = float(F.cosine_similarity(out[:4].double(), ref.double(), dim=-1).min())
        fwd_ms = float(np.median(te))
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            engine()
            torch.cuda.synchronize()
        cls_us = {}
        for e in prof.key_averages():
            t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            if e.key.startswith(("Memcpy", "Memset")) or t <= 0:
                continue
            c = kernel_class(e.key)
            cls_us[c] = cls_us.get(c, 0.0) + t
        total = sum(cls_us.values())
        W, hp, N = ev["width"], math.ceil(ev["mlp"] / 64) * 64, G * G + 1
        gemm_flops = 2 * N * (3 * W * W + W * W + 2 * hp * W + hp * W) * B * ev["layers"]
        r = {"engine_ms": fwd_ms, "torch_bf16_sdpa_ms": float(np.median(tr)), "torch_batch": tb,
             "engine_img_s": B / fwd_ms * 1e3, "min_cosine_vs_fp32": cos_min,
             "layer_gemm_TFLOP_s_over_forward": gemm_flops / fwd_ms / 1e9,
             "kernel_share": {c: us / total for c, us in sorted(cls_us.items())}}
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
