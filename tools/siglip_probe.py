"""Dev probe for the SigLIP models, not a bench line.  Needs a GPU; prints JSON lines.

  1. image forward, device-resident uint8 batch of 256 at the model's size (seeded weights), for ViT-B-16-SigLIP at 224
     and 384 and ViT-L-16-SigLIP-256, beside the engine's own open_clip/ViT-B-16 CLIP image forward at b256 in the same
     process, and transformers' bf16 SiglipVisionModel (SDPA attention) on the same shapes as a yardstick;
  2. the MAP head alone: the kernels the image forward launches after its last block (final LayerNorm over every token,
     K|V GEMM, MAP attention, proj, LayerNorm, fc1, fc2, L2), summed from one torch.profiler trace of a b256 forward,
     over the sum of every kernel of that forward;
  3. text forward, ids on the device, b256 x 64 and b1 x 64 (the single query replays a CUDA graph).
Forward times are host clocks around `iters` calls that end in a device synchronise, after `warmup` calls.

    python tools/siglip_probe.py [iters]
"""
import json
import subprocess
import sys
import time

import torch

sys.path.insert(0, ".")
from marqo_b200 import model_registry as R, weights as Wt  # noqa: E402
from marqo_b200.engine import Encoder  # noqa: E402

ITERS = int(sys.argv[1]) if len(sys.argv) > 1 else 20
WARMUP = 3
MAP_HEAD_KERNELS = 8   # model.cu map_head: layernorm, gemm, map_attention, gemm, layernorm, gemm, gemm, l2_rows


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in q.split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def _wall(fn, iters=ITERS):
    for _ in range(WARMUP):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / iters * 1e3


def _vision_encoder(name):
    arch = dict(R.get_model_properties(name)["arch"], text=None)
    kind = arch.get("kind", "clip")
    sd = (Wt.random_siglip_weights if kind == "siglip" else Wt.random_clip_weights)(arch, 1234)
    return Encoder(kind, arch, sd, max_batch=256), arch


def image(name, B=256, profile_head=False):
    enc, arch = _vision_encoder(name)
    S = arch["vision"]["image_size"]
    imgs = torch.randint(0, 256, (B, S, S, 3), dtype=torch.uint8, device="cuda")
    out = torch.empty((B, enc.embed_dim), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()

    def run():
        enc.encode_images_u8_device(imgs.data_ptr(), B, S, S, out.data_ptr(), sync=True)

    ms = _wall(run)
    rec = {"probe": "image", "model": name, "B": B, "S": S, "ms": ms, "images_per_s": B / ms * 1e3}
    if profile_head:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run()
        ev = sorted((e for e in prof.events() if e.device_type.name == "CUDA" and e.device_time_total > 0),
                    key=lambda e: e.time_range.start)
        total = sum(e.device_time_total for e in ev)
        head = ev[-MAP_HEAD_KERNELS:]
        assert "map_attention" in head[2].name, [e.name for e in head]
        head_us = sum(e.device_time_total for e in head)
        rec.update(kernel_us=total, map_head_us=head_us, map_head_share=head_us / total,
                   map_head_kernels={e.name[:60]: e.device_time_total for e in head})
    enc.close()
    return rec


def hf_image(name, B=256):
    from transformers import SiglipVisionConfig, SiglipVisionModel
    v = R.get_model_properties(name)["arch"]["vision"]
    cfg = SiglipVisionConfig(hidden_size=v["width"], intermediate_size=v["mlp"], num_hidden_layers=v["layers"],
                             num_attention_heads=v["heads"], image_size=v["image_size"], patch_size=v["patch"],
                             hidden_act="gelu", layer_norm_eps=1e-6)
    cfg._attn_implementation = "sdpa"
    model = SiglipVisionModel(cfg).to("cuda", torch.bfloat16).eval()
    S = v["image_size"]
    px = torch.randn(B, 3, S, S, device="cuda", dtype=torch.bfloat16)
    with torch.no_grad():
        ms = _wall(lambda: model(pixel_values=px).pooler_output)
    del model
    torch.cuda.empty_cache()
    return {"probe": "transformers_bf16_sdpa_image", "model": name, "B": B, "S": S, "ms": ms,
            "images_per_s": B / ms * 1e3}


def text(name, B):
    arch = dict(R.get_model_properties(name)["arch"], vision=None)
    enc = Encoder("siglip", arch, Wt.random_siglip_weights(arch, 1234), max_batch=256)
    ids = torch.randint(0, 32000, (B, 64), dtype=torch.int32, device="cuda")
    out = torch.empty((B, enc.embed_dim), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    ms = _wall(lambda: enc.encode_tokens_device(ids.data_ptr(), None, B, 64, out.data_ptr(), sync=True))
    enc.close()
    return {"probe": "text", "model": name, "B": B, "seq": 64, "ms": ms, "texts_per_s": B / ms * 1e3}


def main():
    print(json.dumps(_card()), flush=True)
    b16 = "open_clip/ViT-B-16-SigLIP/webli"
    for _ in range(2):   # the two forwards the 5 % target compares, alternated
        print(json.dumps(image("open_clip/ViT-B-16/laion2b_s34b_b88k")), flush=True)
        print(json.dumps(image(b16)), flush=True)
    print(json.dumps(image(b16, profile_head=True)), flush=True)
    for name in ("open_clip/ViT-B-16-SigLIP-384/webli", "open_clip/ViT-L-16-SigLIP-256/webli"):
        print(json.dumps(image(name, profile_head=True)), flush=True)
    for B in (256, 1):
        print(json.dumps(text(b16, B)), flush=True)
    for name in (b16, "open_clip/ViT-B-16-SigLIP-384/webli", "open_clip/ViT-L-16-SigLIP-256/webli"):
        print(json.dumps(hf_image(name)), flush=True)


if __name__ == "__main__":
    main()
