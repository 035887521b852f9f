"""Images of mixed sizes on one GPU, for ViT-B-32 and ViT-L-14 image towers with seeded weights (no downloads), each
as images/s:

  1. 256 images whose sizes are drawn (seeded) from photo sizes between 480 x 640 and 3000 x 4000, host uint8 arrays:
     through B200OpenCLIP.encode_image's per-size loop (one tower pass per distinct size) and through one
     Encoder.encode_images_u8_ragged call (one resize pass and one tower pass per sub-batch);
  2. the ragged resize kernels alone on those images, device-resident (their kernel time in a torch.profiler run);
  3. a uniform batch of 256 images at 480 x 640 through b200_debug_resize with this build's kernels and, given
     --baseline-lib (another build of libmarqo_b200.so, e.g. the parent commit's), with that build's, alternated in
     one process: the end-to-end call (CUDA events) and the kernels' time (torch.profiler).

Medians over --steps calls after --warmup.  Also prints the card's name and power limit, read in the same process.

    python tools/ragged_probe.py [--steps 5] [--warmup 1] [--models b32,l14] [--baseline-lib PATH] [--out FILE]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from marqo_b200 import _native as N  # noqa: E402
from marqo_b200 import model_registry as R  # noqa: E402
from marqo_b200.engine import Encoder  # noqa: E402
from marqo_b200.loaders import B200OpenCLIP  # noqa: E402
from marqo_b200.weights import random_weights  # noqa: E402

B = 256
NAMES = {"b32": "open_clip/ViT-B-32/laion2b_s34b_b79k", "l14": "open_clip/ViT-L-14/laion2b_s32b_b82k"}
PHOTO_SIZES = [(480, 640), (640, 480), (720, 1280), (768, 1024), (1024, 768), (1080, 1920), (1200, 1600),
               (1536, 2048), (2448, 3264), (3000, 4000), (4000, 3000)]


def median(xs):
    return float(np.median(xs))


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(steps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t)
    return median(ts)


def resize_kernels_ms(fn, tag=None):
    """Device time of the resample kernels one call of fn runs (those whose name contains tag, if given)."""
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    us = sum(e.time_range.elapsed_us() for e in prof.events()
             if e.device_type == DeviceType.CUDA and "resample_" in e.name and (tag is None or tag in e.name))
    return us / 1e3


def ragged_resize(lib, tensors, S, out, stream):
    n = len(tensors)
    ptrs = (C.c_void_p * n)(*[t.data_ptr() for t in tensors])
    hs = np.array([t.shape[0] for t in tensors], np.int32)
    ws = np.array([t.shape[1] for t in tensors], np.int32)
    N.check(lib.b200_debug_resize_ragged(0, ptrs, hs.ctypes.data_as(C.c_void_p), ws.ctypes.data_as(C.c_void_p), n, S,
                                         0, C.c_void_p(out.data_ptr()), C.c_void_p(stream)))


def uniform_resize(lib, batch, S, out, stream):
    n, h, w, _ = batch.shape
    status = lib.b200_debug_resize(0, C.c_void_p(batch.data_ptr()), n, h, w, S, C.c_void_p(out.data_ptr()),
                                   C.c_void_p(stream))
    if status != N.OK:
        raise RuntimeError(f"b200_debug_resize failed: {status}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--models", default="b32,l14")
    ap.add_argument("--baseline-lib")
    ap.add_argument("--out")
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("card:", q, flush=True)
    res = {"card": q, "batch": B, "models": {}}
    lib = N.load()
    stream = torch.cuda.current_stream().cuda_stream

    rng = np.random.default_rng(0)
    sizes = [PHOTO_SIZES[i] for i in rng.integers(0, len(PHOTO_SIZES), B)]
    pool = {s: rng.integers(0, 256, s + (3,), dtype=np.uint8) for s in set(sizes)}   # one pixel block per size
    imgs = [pool[s] for s in sizes]
    res["distinct_sizes"] = len(pool)
    res["source_mb"] = sum(a.nbytes for a in imgs) / 1e6

    for key in args.models.split(","):
        arch = R.get_model_properties(NAMES[key])["arch"]
        arch["text"] = None
        enc = Encoder("clip", arch, random_weights("clip", arch, 1), max_batch=B)
        loader = B200OpenCLIP.__new__(B200OpenCLIP)
        loader.model = enc
        r = {}
        per_size = timed(lambda: loader.encode_image(imgs), args.steps, args.warmup)
        ragged = timed(lambda: enc.encode_images_u8_ragged(imgs), args.steps, args.warmup)
        same = np.array_equal(loader.encode_image(imgs), enc.encode_images_u8_ragged(imgs))
        r["mixed_per_size_loop_img_s"] = B / per_size
        r["mixed_ragged_img_s"] = B / ragged
        r["mixed_speedup"] = per_size / ragged
        r["mixed_rows_equal"] = bool(same)   # the per-size loop runs other batch sizes: equal bits are not promised
        res["models"][key] = r
        print(key, json.dumps(r), flush=True)
        enc.close()

    dev = {s: torch.from_numpy(a).cuda() for s, a in pool.items()}
    tensors = [dev[s] for s in sizes]
    out = torch.empty((B, 224, 224, 3), dtype=torch.uint8, device="cuda")
    ragged_resize(lib, tensors, 224, out, stream)
    ms = [resize_kernels_ms(lambda: ragged_resize(lib, tensors, 224, out, stream)) for _ in range(args.steps)]
    res["mixed_resize_kernels_ms"] = median(ms)
    res["mixed_resize_kernels_img_s"] = B / (median(ms) / 1e3)
    print("mixed resize kernels:", median(ms), "ms", flush=True)
    del dev, tensors

    batch = torch.from_numpy(np.random.default_rng(1).integers(0, 256, (B, 480, 640, 3), dtype=np.uint8)).cuda()
    libs = {"new": lib}
    if args.baseline_lib:
        base = C.CDLL(os.path.abspath(args.baseline_lib))
        base.b200_debug_resize.restype = C.c_int
        base.b200_debug_resize.argtypes = lib.b200_debug_resize.argtypes
        libs["baseline"] = base
    outs = {k: torch.empty((B, 224, 224, 3), dtype=torch.uint8, device="cuda") for k in libs}
    for k, L in libs.items():
        uniform_resize(L, batch, 224, outs[k], stream)
    if "baseline" in libs:
        res["uniform_outputs_equal"] = bool(torch.equal(outs["new"], outs["baseline"]))
    call = {k: [] for k in libs}
    kern = {k: [] for k in libs}
    for _ in range(args.steps):
        for k, L in libs.items():   # alternated
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            uniform_resize(L, batch, 224, outs[k], stream)
            e.record()
            e.synchronize()
            call[k].append(s.elapsed_time(e))
            kern[k].append(resize_kernels_ms(lambda: uniform_resize(L, batch, 224, outs[k], stream),
                                             "ResizeDesc" if k == "new" else None))
    for k in libs:
        res[f"uniform_{k}_call_ms"] = median(call[k])
        res[f"uniform_{k}_kernels_ms"] = median(kern[k])
        res[f"uniform_{k}_kernels_img_s"] = B / (median(kern[k]) / 1e3)
    print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
