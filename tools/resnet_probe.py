"""ResNet CLIP image forwards on one GPU: the engine's RN50 and RN101 at b256 (device-resident uint8 at 224) against
torch running the oracle network (tests/_resnet_oracle.py, as nn modules via cuDNN) under fp16 autocast in NCHW -- what
the reference runs on CUDA -- and under bf16 channels_last, alternated in one process.  Prints the card and its power
limit, the engine's GEMM-class share (b200_model_profile) and the achieved TFLOP/s of every conv shape (FLOPs from
shapes, kernel time from torch.profiler over the launches of that shape).

    python tools/resnet_probe.py [--steps 20] [--warmup 3] [--out FILE]

The results are printed; --out also writes them to FILE as JSON."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import _resnet_oracle as O  # noqa: E402
from marqo_b200 import model_registry as R  # noqa: E402
from marqo_b200.engine import Encoder  # noqa: E402
from marqo_b200.weights import random_clip_resnet_weights  # noqa: E402

B, S = 256, 224


def conv_flops(arch, n):
    """[(label, flops)] of every conv / GEMM of the image forward in launch order (2 * M * N * K)."""
    r, E = arch["resnet"], arch["embed_dim"]
    w, out = r["width"], []
    H = S // 2
    out += [(f"stem 3->{w // 2} s2", 2 * n * H * H * (w // 2) * 27), (f"3x3 {w // 2}->{w // 2} @{H}", 2 * n * H * H * (w // 2) * 9 * (w // 2)),
            (f"3x3 {w // 2}->{w} @{H}", 2 * n * H * H * w * 9 * (w // 2))]
    H //= 2
    inplanes = w
    for s, depth in enumerate(r["layers"]):
        planes = w << s
        for i in range(depth):
            stride = 2 if (i == 0 and s > 0) else 1
            out.append((f"1x1 {inplanes}->{planes} @{H}", 2 * n * H * H * planes * inplanes))
            out.append((f"3x3 {planes}->{planes} @{H}", 2 * n * H * H * planes * 9 * planes))
            H //= stride
            if i == 0:
                out.append((f"1x1 {inplanes}->{4 * planes} @{H} (ds)", 2 * n * H * H * 4 * planes * inplanes))
            out.append((f"1x1 {planes}->{4 * planes} @{H}", 2 * n * H * H * 4 * planes * planes))
            inplanes = 4 * planes
    C, T = inplanes, H * H + 1
    out += [("attnpool k|v", 2 * n * T * 2 * C * C), ("attnpool q", 2 * n * C * C), ("attnpool c_proj", 2 * n * E * C)]
    return out


class TorchNet(torch.nn.Module):
    def __init__(self, sd, arch):
        super().__init__()
        self.sd = {k: torch.as_tensor(v).float().cuda() for k, v in sd.items() if k.startswith("visual.")}
        self.arch = arch

    def forward(self, x):
        y = O.attnpool(self.sd, O.trunk(self.sd, self.arch["resnet"]["layers"], x), self.arch["resnet"]["heads"])
        return y / y.norm(dim=-1, keepdim=True)


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the results to this JSON file")
    a = ap.parse_args()
    torch.backends.cudnn.benchmark = True
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card)
    rng = np.random.default_rng(0)
    imgs = torch.from_numpy(rng.integers(0, 256, (B, S, S, 3), dtype=np.uint8)).cuda()
    mean = torch.tensor(R.OPENAI_MEAN, device="cuda").view(1, 3, 1, 1)
    std = torch.tensor(R.OPENAI_STD, device="cuda").view(1, 3, 1, 1)
    pix = ((imgs.permute(0, 3, 1, 2).float() / 255.0) - mean) / std
    res = {"card": card, "batch": B, "models": {}}
    models = {}
    for name in ("open_clip/RN50/openai", "open_clip/RN101/openai"):
        arch = R.get_model_properties(name)["arch"]
        arch["layers"] = 0
        sd = random_clip_resnet_weights(arch, seed=1)
        enc = Encoder("clip_resnet", arch, sd, max_batch=B)
        out = torch.empty((B, arch["embed_dim"]), dtype=torch.float32, device="cuda")
        net = TorchNet(sd, arch)
        net_cl = TorchNet(sd, arch)
        net_cl.sd = {k: (v.to(memory_format=torch.channels_last) if v.dim() == 4 else v) for k, v in net.sd.items()}
        models[name] = (arch, enc, out, net, net_cl)
    timings = {n: {"engine": [], "torch_fp16_nchw": [], "torch_bf16_cl": []} for n in models}
    pix_cl = pix.contiguous(memory_format=torch.channels_last)
    for _, enc, _, _, _ in models.values():   # the engine on torch's stream, so that the CUDA events time its work
        enc.set_stream(torch.cuda.current_stream().cuda_stream)
    for rep in range(2):   # the models and the three runs alternated
        for name, (arch, enc, out, net, net_cl) in models.items():
            eng = lambda: enc.encode_images_u8_device(imgs.data_ptr(), B, S, S, out.data_ptr(), sync=False)
            torch.cuda.synchronize()
            timings[name]["engine"].append(_time(eng, a.steps, a.warmup))
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
                timings[name]["torch_fp16_nchw"].append(_time(lambda: net(pix), a.steps, a.warmup))
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                timings[name]["torch_bf16_cl"].append(_time(lambda: net_cl(pix_cl), a.steps, a.warmup))
    for name, (arch, enc, out, net, net_cl) in models.items():
        enc.set_stream(None)
        enc.set_profiling(True)   # GEMM-class vs attention-class device time of one forward
        enc.encode_images_u8_device(imgs.data_ptr(), B, S, S, out.data_ptr(), sync=True)
        prof = enc.profile()
        enc.set_profiling(False)
        # per-conv kernel time: torch.profiler's CUDA activity of one forward; the GEMM kernels run in conv_flops order
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as tp:
            enc.encode_images_u8_device(imgs.data_ptr(), B, S, S, out.data_ptr(), sync=True)
        kern = sorted((e for e in tp.events() if e.device_type.name == "CUDA" and "gemm" in e.name),
                      key=lambda e: e.time_range.start)
        flops = conv_flops(arch, B)
        per_shape = {}
        if len(kern) == len(flops):
            for (label, f), e in zip(flops, kern):
                d = per_shape.setdefault(label, {"flops": 0, "us": 0.0, "launches": 0})
                d["flops"] += f
                d["us"] += e.time_range.elapsed_us()
                d["launches"] += 1
            for d in per_shape.values():
                d["tflops"] = d["flops"] / (d["us"] * 1e-6) / 1e12
        else:
            print(f"{name}: {len(kern)} GEMM kernels for {len(flops)} convs: per-shape rates not attributed")
        total_fl = sum(f for _, f in flops)
        r = {"engine_ms": timings[name]["engine"], "torch_fp16_nchw_ms": timings[name]["torch_fp16_nchw"],
             "torch_bf16_channels_last_ms": timings[name]["torch_bf16_cl"], "profile": prof,
             "gemm_share_of_forward": prof["gemm_ms"] / float(np.median(timings[name]["engine"])),
             "gemm_tflops_avg": total_fl / (prof["gemm_ms"] * 1e-3) / 1e12, "per_shape": per_shape}
        res["models"][name] = r
        print(json.dumps({name: {k: v for k, v in r.items() if k != "per_shape"}}))
        for label, d in per_shape.items():
            print(f"  {label:32s} {d['launches']:3d} launches {d['us']:9.1f} us {d['tflops']:7.1f} TFLOP/s")
        enc.close()
    if a.out is None:
        return
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
