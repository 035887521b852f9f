"""Dev probe: mean device time of the GEMM kernel alone, per shape and epilogue (not a bench line).  Needs a GPU; prints
the card, then one JSON line per case.

Default cases are the four ViT-L-14 layer GEMMs of the headline step (M = 256 images x 257 tokens), first with the
epilogue the encoder runs them with, then with the plain epilogue (bf16 output, no bias, no residual): the difference
is what the epilogue costs.  Each line also times torch.matmul in bf16 at the same M, N, K (CUDA events, same
iteration count) as a yardstick for the main loop.

    python tools/gemm_probe.py [iters]
    python tools/gemm_probe.py M N K act out_bf16 has_bias residual_in_place [iters]
"""
import ctypes as C
import json
import subprocess
import sys

import torch

sys.path.insert(0, ".")
from marqo_b200 import _native as N  # noqa: E402

M = 256 * 257
GELU = 1
# name, N, K, act, out_bf16, has_bias, residual_in_place
LAYER = [
    ("qkv", 3072, 1024, 0, 1, 1, 0),
    ("out_proj", 1024, 1024, 0, 0, 1, 1),
    ("fc1", 4096, 1024, GELU, 1, 1, 0),
    ("fc2", 1024, 4096, 0, 0, 1, 1),
]


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in q.split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def _torch_ms(m, n, k, iters):
    a = torch.randn(m, k, device="cuda", dtype=torch.bfloat16)
    w = torch.randn(n, k, device="cuda", dtype=torch.bfloat16)
    for _ in range(3):
        torch.matmul(a, w.t())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        torch.matmul(a, w.t())
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    args = [int(x) for x in sys.argv[1:]]
    if len(args) >= 7:
        m = args[0]
        cases = [("custom", *args[1:7])]
        iters = args[7] if len(args) > 7 else 20
    else:
        m = M
        iters = args[0] if args else 20
        cases = LAYER + [(name + "_plain", n, k, 0, 1, 0, 0) for name, n, k, *_ in LAYER]
    print(json.dumps(_card()), flush=True)
    lib = N.load()
    for name, n, k, act, out_bf16, has_bias, res in cases:
        ms = C.c_float(0)
        N.check(lib.b200_debug_gemm_time(0, m, n, k, act, out_bf16, has_bias, res, iters, C.byref(ms)))
        flops = 2.0 * m * n * k
        tms = _torch_ms(m, n, k, iters)
        print(json.dumps({"case": name, "M": m, "N": n, "K": k, "act": act, "out_bf16": out_bf16,
                          "bias": has_bias, "residual_in_place": res, "us": round(ms.value * 1e3, 1),
                          "TFLOPs": round(flops / ms.value / 1e9, 1), "torch_bf16_us": round(tms * 1e3, 1),
                          "torch_TFLOPs": round(flops / tms / 1e9, 1)}), flush=True)


if __name__ == "__main__":
    main()
