"""The wide OpenAI ResNet CLIP image towers (RN50x16 at 384 px, RN50x64 at 448 px) on one GPU, at the `clip` loader's
default batch (loaders.WIDE_RESNET_MAX_BATCH) of device-resident uint8 images at the model's size: images/s, the
device bytes the model holds (b200_debug_device_bytes), and the kernel time of every conv shape (torch.profiler over
one forward's GEMM launches) beside torch's own bf16 channels-last conv2d of that shape (CUDA events).  Prints the
card and its power limit.

    python tools/openai_clip_probe.py [--steps 10] [--warmup 2] [--out FILE]

The results are printed; --out also writes them to FILE as JSON."""
import argparse
import copy
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from marqo_b200 import _native as N, model_registry as R  # noqa: E402
from marqo_b200.engine import Encoder  # noqa: E402
from marqo_b200.loaders import WIDE_RESNET_MAX_BATCH as B  # noqa: E402
from marqo_b200.weights import random_clip_resnet_weights  # noqa: E402


def convs(arch):
    """[(label, (cin, cout, k, H))] of every conv of the image forward in launch order (H: output side), then the
    attention pool's three GEMMs (label only)."""
    r = arch["resnet"]
    w, S = r["width"], r["image_size"]
    H = S // 2
    out = [(f"stem 3->{w // 2} s2", (3, w // 2, 3, H)), (f"3x3 {w // 2}->{w // 2} @{H}", (w // 2, w // 2, 3, H)),
           (f"3x3 {w // 2}->{w} @{H}", (w // 2, w, 3, H))]
    H //= 2
    inplanes = w
    for s, depth in enumerate(r["layers"]):
        planes = w << s
        for i in range(depth):
            stride = 2 if (i == 0 and s > 0) else 1
            out.append((f"1x1 {inplanes}->{planes} @{H}", (inplanes, planes, 1, H)))
            out.append((f"3x3 {planes}->{planes} @{H}", (planes, planes, 3, H)))
            H //= stride
            if i == 0:
                out.append((f"1x1 {inplanes}->{4 * planes} @{H} (ds)", (inplanes, 4 * planes, 1, H)))
            out.append((f"1x1 {planes}->{4 * planes} @{H}", (planes, 4 * planes, 1, H)))
            inplanes = 4 * planes
    return out + [("attnpool k|v", None), ("attnpool q", None), ("attnpool c_proj", None)]


def _time(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(steps):
        fn()
    ev1.record()
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1) / steps


def torch_conv_us(shape, n, steps, warmup):
    """torch bf16 channels-last conv2d of one conv shape over n images (the stem with stride 2)."""
    cin, cout, k, H = shape
    Hin = 2 * H if cin == 3 else H
    x = torch.randn(n, cin, Hin, Hin, device="cuda", dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    w = torch.randn(cout, cin, k, k, device="cuda", dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    f = lambda: torch.nn.functional.conv2d(x, w, stride=2 if cin == 3 else 1, padding=k // 2)
    return 1e3 * _time(f, steps, warmup)


def device_bytes():
    n = C.c_int64()
    N.check(N.load().b200_debug_device_bytes(C.byref(n)))
    return n.value


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the results to this JSON file")
    a = ap.parse_args()
    torch.backends.cudnn.benchmark = True
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card)
    res = {"card": card, "batch": B, "models": {}}
    for name in ("RN50x16", "RN50x64"):
        arch = copy.deepcopy(R.WIDE_RESNET_ARCHS[name])   # (served from custom checkpoints: not registry names)
        arch["layers"] = 0   # the image tower alone
        S = arch["resnet"]["image_size"]
        sd = random_clip_resnet_weights(arch, seed=1)
        before = device_bytes()
        enc = Encoder("clip_resnet", arch, sd, max_batch=B)
        held = device_bytes() - before
        imgs = torch.from_numpy(np.random.default_rng(0).integers(0, 256, (B, S, S, 3), dtype=np.uint8)).cuda()
        out = torch.empty((B, arch["embed_dim"]), dtype=torch.float32, device="cuda")
        enc.set_stream(torch.cuda.current_stream().cuda_stream)   # the CUDA events time the engine's work
        fwd = lambda: enc.encode_images_u8_device(imgs.data_ptr(), B, S, S, out.data_ptr(), sync=False)
        ms = [_time(fwd, a.steps, a.warmup) for _ in range(2)]
        enc.set_stream(None)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as tp:
            enc.encode_images_u8_device(imgs.data_ptr(), B, S, S, out.data_ptr(), sync=True)
        kern = sorted((e for e in tp.events() if e.device_type.name == "CUDA" and "gemm" in e.name),
                      key=lambda e: e.time_range.start)
        plan = convs(arch)
        per_shape = {}
        if len(kern) == len(plan):
            for (label, shape), e in zip(plan, kern):
                d = per_shape.setdefault(label, {"shape": shape, "us": 0.0, "launches": 0})
                d["us"] += e.time_range.elapsed_us()
                d["launches"] += 1
            for d in per_shape.values():
                d["engine_us_per_launch"] = d["us"] / d["launches"]
                if d["shape"] is not None:
                    d["torch_bf16_cl_us"] = torch_conv_us(d["shape"], B, a.steps, a.warmup)
        else:
            print(f"{name}: {len(kern)} GEMM kernels for {len(plan)} GEMMs: per-shape times not attributed")
        r = {"image_size": S, "forward_ms": ms, "images_per_s": B / (min(ms) * 1e-3), "device_bytes": held,
             "per_shape": per_shape}
        res["models"][name] = r
        print(json.dumps({name: {k: v for k, v in r.items() if k != "per_shape"}}))
        for label, d in per_shape.items():
            t = d.get("torch_bf16_cl_us")
            print(f"  {label:34s} {d['launches']:3d} x {d['engine_us_per_launch']:9.1f} us"
                  + (f"   torch bf16 channels-last {t:9.1f} us" if t is not None else ""))
        enc.close()
        del imgs, out
        torch.cuda.empty_cache()
    if a.out is None:
        return
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
