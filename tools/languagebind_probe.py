"""Speed of LanguageBind/Video_V1.5_FT's video encode on the engine (seeded weights, the full ViT-L/14 video tower of
24 layers over 8 frames), printed as one JSON line per measurement:

  - videos/s of encode_videos_u8 at n = 1, 8 and 32 (uint8 frames of --height x --width, host in, host out; the
    host clock around calls that end in a device synchronise, after warm-up);
  - GEMM and attention device time of one n = 8 call from b200_model_profile (the temporal attention counts as
    attention), and the share of the temporal kernels (temporal_embed_ln, temporal_attention) in the call's kernel
    time from torch.profiler, in a run of its own;
  - the same forward (n = 8, transformed frames in) in torch under bf16 autocast with SDPA, over this repository's
    fp32 restatement of the reference module (tests/_languagebind_oracle.py);
  - temporal_attention alone at n = 8: its algorithmic bytes (q, k, v read once, the output written once) over its
    kernel time, against the H100 SXM's 3.35 TB/s.

The card's name and power limit are read in the same run.  Nothing is written unless --out is given.

Run:  python tools/languagebind_probe.py [--out languagebind_probe.json]
"""
import argparse
import copy
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

from marqo_b200 import engine as E  # noqa: E402
from marqo_b200 import model_registry as R  # noqa: E402
from marqo_b200 import weights as W  # noqa: E402

NAME = "LanguageBind/Video_V1.5_FT"
HBM_TBS = 3.35


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def _time(fn, iters):
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--height", type=int, default=240)
    ap.add_argument("--width", type=int, default=320)
    ap.add_argument("--out")
    args = ap.parse_args()
    card = _card()
    arch = copy.deepcopy(R.LANGUAGEBIND_MODELS[NAME]["arch"])
    T, L = arch["video_frames"], arch["vision"]["layers"]
    sd = W.random_languagebind_video_weights(arch, 1)
    enc = E.Encoder("clip", arch, W.languagebind_video_state_dict_to_engine(sd), max_batch=32)
    rng = np.random.default_rng(0)
    lines = []

    def emit(d):
        d = {"card": card, **d}
        print(json.dumps(d), flush=True)
        lines.append(d)

    for n in (1, 8, 32):
        v = rng.integers(0, 256, (n, T, args.height, args.width, 3), dtype=np.uint8)
        s = _time(lambda: enc.encode_videos_u8(v), 3 if n == 32 else 10)
        emit({"what": "engine encode_videos_u8", "n": n, "ms": s * 1e3, "videos_per_s": n / s})

    v8 = rng.integers(0, 256, (8, T, args.height, args.width, 3), dtype=np.uint8)
    enc.encode_videos_u8(v8)
    enc.set_profiling(True)
    enc.encode_videos_u8(v8)
    prof = enc.profile()
    enc.set_profiling(False)
    call_ms = enc.last_timing()[0]
    emit({"what": "engine profile n=8", "call_ms": call_ms, **prof})

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        enc.encode_videos_u8(v8)
        torch.cuda.synchronize()
    total = temporal = 0.0
    for e in p.key_averages():
        t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        if e.key.startswith(("cudaMemcpy", "Memcpy", "Memset")):
            continue
        total += t
        if "temporal_" in e.key:
            temporal += t
    emit({"what": "temporal kernels' share n=8", "temporal_us": temporal, "kernels_us": total,
          "share": temporal / total if total else None})
    enc.close()

    import _languagebind_oracle as O
    import torch.nn.functional as F

    def sdpa_mha(x, sdx, pfx, heads, causal=False):
        B, Lq, Wd = x.shape
        q, k, vv = (O._lin(x, sdx, pfx + nm + "_proj.").view(B, Lq, heads, Wd // heads).transpose(1, 2)
                    for nm in ("q", "k", "v"))
        o = F.scaled_dot_product_attention(q, k, vv, is_causal=causal).transpose(1, 2).reshape(B, Lq, Wd)
        return O._lin(o, sdx, pfx + "out_proj.")

    O._mha = sdpa_mha
    sdc = {k: torch.from_numpy(np.asarray(a, np.float32)).cuda() for k, a in sd.items()}
    px = torch.randn(8, T, 3, 224, 224, device="cuda")
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        s = _time(lambda: O.video_pooled(sdc, px, arch["vision"]["heads"], arch["act"], L), 3)
    emit({"what": "torch bf16 autocast + SDPA, oracle restatement", "n": 8, "ms": s * 1e3, "videos_per_s": 8 / s})

    n, N, Wd, H = 8, 257, arch["vision"]["width"], arch["vision"]["heads"]
    ms = E.debug_temporal_attention_time(n, T, N, Wd, H, iters=50)
    nbytes = n * T * N * (3 * Wd + Wd) * 2
    emit({"what": "temporal_attention n=8", "kernel_us": ms * 1e3, "bytes": nbytes,
          "tb_per_s": nbytes / (ms * 1e-3) / 1e12, "share_of_3.35TBs": nbytes / (ms * 1e-3) / 1e12 / HBM_TBS})
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
