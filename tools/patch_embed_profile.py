"""Dev probe: device time of the ViT patch embedding (the gather GEMM and the token-row fill kernel before it) in the
b256 image forward of ViT-L-14 and ViT-B-32, from a torch.profiler trace with CUDA activities.  One JSON line per
model: mean µs per forward of each kernel, over `iters` profiled forwards after two warm-up ones.

    python tools/patch_embed_profile.py [iters]

MARQO_B200_LIB=<path> profiles another build of the library (the kernel names are matched by prefix, so an older
build's fill kernel is reported under its own name)."""
import json
import sys

import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, ".")
from marqo_b200 import model_registry as R, weights as Wt  # noqa: E402
from marqo_b200.engine import Encoder  # noqa: E402

MODELS = ["open_clip/ViT-L-14/laion2b_s32b_b82k", "open_clip/ViT-B-32/laion2b_s34b_b79k"]
B = 256
iters = int(sys.argv[1]) if len(sys.argv) > 1 else 10
torch.cuda.set_device(0)
for name in MODELS:
    arch = dict(R.get_model_properties(name)["arch"])
    arch["text"] = None
    enc = Encoder("clip", arch, Wt.random_clip_weights(arch, 1234), max_batch=B)
    g = torch.Generator(device="cuda").manual_seed(0)
    img = torch.randint(0, 256, (B, 224, 224, 3), dtype=torch.uint8, device="cuda", generator=g)
    out = torch.empty(B, enc.embed_dim, dtype=torch.float32, device="cuda")
    run = lambda: enc.encode_images_u8_device(img.data_ptr(), B, 224, 224, out.data_ptr())
    for _ in range(2):
        run()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            run()
        torch.cuda.synchronize()
    us = {}
    for ev in prof.key_averages():
        # the patch-embed GEMM is the only gemm_kernel instantiation with GATHER = true
        if ev.key.startswith(("void mb::gemm::gemm_kernel<true", "mb::kernels::vit_", "void mb::kernels::vit_")):
            us[ev.key.split("(")[0]] = round(ev.device_time_total / iters, 1)
    print(json.dumps({"model": name, "B": B, "iters": iters, "us_per_forward": us,
                      "patch_embed_us": round(sum(us.values()), 1)}), flush=True)
    enc.close()
