"""OWL-ViT reranking speed on one GPU: the engine's detect call against transformers' OwlViTForObjectDetection, with
seeded weights, over 10 and 50 hits of 240 x 240 images, for B/32, B/16 and L/14.

  engine       Encoder.detect_images_u8: one call for all the hits (squash, trunk, heads, text tower)
  hf_fp32_1x1  the reference's way: fp32, one image per forward (query repeated), eager attention
  hf_bf16_sdpa batched under bf16 autocast with SDPA attention

Prints one JSON line per (model, hits) with median milliseconds, the engine's GEMM and attention shares of one call
(b200_model_profile) and the card's name and power limit; with --out FILE, also writes them all there as JSON."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


def _card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def _median_ms(fn, reps: int) -> float:
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(times))


def _hf(arch, sd, attn):
    import transformers
    v, t = arch["vision"], arch["text"]
    cfg = transformers.OwlViTConfig(
        text_config={"hidden_size": t["width"], "num_hidden_layers": t["layers"], "num_attention_heads": t["heads"],
                     "intermediate_size": t["mlp"], "vocab_size": t["vocab"], "max_position_embeddings": 16},
        vision_config={"hidden_size": v["width"], "num_hidden_layers": v["layers"], "num_attention_heads": v["heads"],
                       "intermediate_size": v["mlp"], "patch_size": v["patch"], "image_size": v["image_size"]},
        projection_dim=arch["embed_dim"], attn_implementation=attn)
    m = transformers.OwlViTForObjectDetection(cfg).eval()
    own = m.state_dict()
    fixed = {(k.replace("pre_layrnorm", "pre_layernorm") if k not in own else k): torch.from_numpy(np.asarray(x))
             for k, x in sd.items()}
    m.load_state_dict({k: x.reshape(own[k].shape) for k, x in fixed.items()}, strict=False)
    return m.cuda()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="owl/ViT-B/32,owl/ViT-B/16,owl/ViT-L/14")
    ap.add_argument("--hits", default="10,50")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from marqo_b200 import model_registry as R, weights as W
    from marqo_b200.engine import Encoder
    card = _card()
    rows = []
    ids = np.zeros(16, np.int32)
    ids[:6] = [49406, 320, 1929, 539, 320, 49407]
    for name in a.models.split(","):
        arch = R.OWL_VIT_MODELS[name]["arch"]
        sd = W.random_owlvit_weights(arch, 1)
        enc = Encoder("clip", arch, W.owlvit_state_dict_to_engine(sd), max_batch=32)
        S = arch["vision"]["image_size"]
        for n in (int(x) for x in a.hits.split(",")):
            imgs = np.random.default_rng(n).integers(0, 256, (n, 240, 240, 3), dtype=np.uint8)
            for _ in range(2):
                enc.detect_images_u8(imgs, ids)
            eng = _median_ms(lambda: enc.detect_images_u8(imgs, ids), a.reps)
            enc.set_profiling(True)
            enc.detect_images_u8(imgs, ids)
            prof = enc.profile()
            enc.set_profiling(False)
            # HF inputs at the model's size: the squash itself is not timed on either side
            px = torch.randn(n, 3, S, S, device="cuda")
            q = torch.from_numpy(ids).long().cuda()[None]
            res = {"model": name, "hits": n, "engine_ms": eng, "gemm_ms": prof["gemm_ms"],
                   "attention_ms": prof["attention_ms"], "card": card}
            with torch.no_grad():
                m = _hf(arch, sd, "eager")
                one = lambda: [m(input_ids=q, pixel_values=px[i:i + 1], attention_mask=(q != 0).long())
                               for i in range(n)]
                one()
                res["hf_fp32_1x1_ms"] = _median_ms(one, max(1, a.reps // 2))
                del m
                m = _hf(arch, sd, "sdpa")
                qq = q.expand(n, 16)
                bat = lambda: m(input_ids=qq, pixel_values=px, attention_mask=(qq != 0).long())
                with torch.autocast("cuda", dtype=torch.bfloat16):
                    bat()
                    res["hf_bf16_sdpa_ms"] = _median_ms(bat, a.reps)
                del m
                torch.cuda.empty_cache()
            print(json.dumps(res), flush=True)
            rows.append(res)
        enc.close()
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(rows, indent=1))


if __name__ == "__main__":
    main()
