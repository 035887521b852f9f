"""ConvNeXt CLIP image forwards on one GPU: the engine's convnext_base_w, convnext_large_d and convnext_xxlarge at
b256 (device-resident uint8 at the model's size) against torch running the oracle (tests/_convnext_oracle.py) under
bf16 autocast in channels_last, the two alternated in one process (3 warm-up and `--steps` timed calls each).  Prints
the card and its power limit, the engine's GEMM-class share (b200_model_profile), and the achieved bytes/s of the three
ConvNeXt kernels (bytes each must move, from shapes, over their kernel time in a torch.profiler run of its own).

    python tools/convnext_probe.py [--steps 20] [--warmup 3] [--models base_w,large_d,xxlarge] [--out FILE]

The results are printed; --out also writes them to FILE as JSON."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import _convnext_oracle as O  # noqa: E402
from marqo_b200 import model_registry as R  # noqa: E402
from marqo_b200.engine import Encoder  # noqa: E402
from marqo_b200.weights import random_clip_convnext_weights  # noqa: E402

B = 256
NAMES = {"base_w": "open_clip/convnext_base_w/laion2b_s13b_b82k",
         "large_d": "open_clip/convnext_large_d/laion2b_s26b_b102k_augreg",
         "xxlarge": "open_clip/convnext_xxlarge/laion2b_s34b_b82k_augreg"}
MEAN = torch.tensor(R.OPENAI_MEAN).view(1, 3, 1, 1)
STD = torch.tensor(R.OPENAI_STD).view(1, 3, 1, 1)


def kernel_bytes(cx, n):
    """{kernel: bytes one forward must move}: fp32 x read once and bf16 written once per dwconv7_ln / ln_pixels
    (fp32 both ways for the stem's), x read once by pool_ln."""
    S, dims, depths = cx["image_size"], cx["dims"], cx["depths"]
    out = {"dwconv7_ln": 0, "ln_pixels": 0, "pool_ln": 0}
    H = S // 4
    out["ln_pixels"] += n * H * H * dims[0] * 8
    for s, (C, d) in enumerate(zip(dims, depths)):
        if s:
            out["ln_pixels"] += n * H * H * dims[s - 1] * 6
            H //= 2
        out["dwconv7_ln"] += d * n * H * H * C * 6
    out["pool_ln"] += n * H * H * dims[3] * 4
    return out


def events_ms(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--models", default="base_w,large_d,xxlarge")
    ap.add_argument("--out")
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    res = {"card": q, "batch": B, "models": {}}
    print("card:", q, flush=True)
    for key in args.models.split(","):
        arch = R.get_model_properties(NAMES[key])["arch"]
        arch["layers"] = 0
        cx, E = arch["convnext"], arch["embed_dim"]
        S = cx["image_size"]
        t0 = time.time()
        sd = random_clip_convnext_weights(arch, seed=1)
        enc = Encoder("clip_convnext", arch, sd, max_batch=B)
        enc.set_stream(torch.cuda.current_stream().cuda_stream)   # the events below time the engine's own launches
        print(f"{key}: weights + finalize {time.time() - t0:.1f} s", flush=True)
        tsd = {k: torch.as_tensor(v).cuda() for k, v in sd.items()}
        del sd
        img = torch.randint(0, 256, (B, S, S, 3), dtype=torch.uint8, device="cuda")
        out = torch.empty((B, E), device="cuda")

        def engine():
            enc.encode_images_u8_device(img.data_ptr(), B, S, S, out.data_ptr(), sync=False)

        def reference():
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                x = ((img.permute(0, 3, 1, 2).float() / 255 - MEAN.cuda()) / STD.cuda())
                O.encode_image(tsd, arch, x.contiguous(memory_format=torch.channels_last))

        for _ in range(args.warmup):
            engine()
            reference()
        torch.cuda.synchronize()
        te, tr = [], []
        for _ in range(args.steps):
            te.append(events_ms(engine))
            tr.append(events_ms(reference))
        # agreement with the fp32 oracle on a few rows
        with torch.no_grad():
            x = (img[:4].permute(0, 3, 1, 2).float() / 255 - MEAN.cuda()) / STD.cuda()
            old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
            torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
            ref = O.encode_image(tsd, arch, x)
            torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old
        cos = float(torch.nn.functional.cosine_similarity(out[:4].double(), ref.double(), dim=-1).min())
        enc.set_profiling(True)
        engine()
        torch.cuda.synchronize()
        p = enc.profile()
        enc.set_profiling(False)
        fwd_ms = float(np.median(te))
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            engine()
            torch.cuda.synchronize()
        kus = {k: 0.0 for k in ("dwconv7_ln", "ln_pixels", "pool_ln")}
        for ev in prof.key_averages():
            for k in kus:
                if k + "_kernel" in ev.key:
                    kus[k] += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        nbytes = kernel_bytes(cx, B)
        r = {"engine_ms": fwd_ms, "torch_bf16_cl_ms": float(np.median(tr)), "engine_img_s": B / fwd_ms * 1e3,
             "min_cosine_vs_fp32_oracle": cos, "gemm_ms_profiled": p["gemm_ms"], "gemm_launches": p["gemm_launches"],
             "gemm_share": p["gemm_ms"] / fwd_ms,
             "kernels": {k: {"us": kus[k], "GB_s": nbytes[k] / (kus[k] * 1e-6) / 1e9 if kus[k] else None,
                             "share": kus[k] / 1e3 / fwd_ms} for k in kus}}
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
