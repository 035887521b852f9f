"""The Stella embedder (Marqo/dunzhang-stella_en_400M_v5, GTE encoder) on one GPU: the engine (device-resident token
ids, seeded weights) against torch running the same weights (the tests' fp32 restatement, tests/_gte_oracle.py, with
the attention through scaled_dot_product_attention) under bf16 autocast, the two alternated in one process
(`--warmup` and `--steps` calls each, medians reported), at three shapes: b256 x 128 tokens, b64 x 512 and a single
16-token query.  Also prints the card's name and power limit, read in the same process, and the share of the engine's
b64 x 512 forward that is neither GEMM nor attention by b200_model_profile (the embedding, LayerNorms, rope, GeGLU and
pooling kernels), with a torch.profiler breakdown of it by kernel (a run of its own).

    python tools/gte_probe.py [--steps 10] [--warmup 2] [--out FILE]

The results are printed; --out also writes them to FILE as JSON."""
import argparse
import json
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

from marqo_b200.engine import Encoder  # noqa: E402
import _gte_oracle as G  # noqa: E402

SHAPES = [("b256x128", 256, 128), ("b64x512", 64, 512), ("b1x16", 1, 16)]


def torch_forward(sd, cfg, ids, mask, cos, sin):
    """tests/_gte_oracle.py's forward with the attention through scaled_dot_product_attention."""
    B, S = ids.shape
    w, H = cfg.width, cfg.heads
    x = sd["embeddings.word_embeddings.weight"][ids] + sd["embeddings.token_type_embeddings.weight"][0]
    x = F.layer_norm(x, (w,), sd["embeddings.LayerNorm.weight"], sd["embeddings.LayerNorm.bias"], cfg.ln_eps)
    keep = mask.bool()[:, None, None, :]
    for i in range(cfg.layers):
        p = f"encoder.layer.{i}."
        q, k, v = F.linear(x, sd[p + "attention.qkv_proj.weight"], sd[p + "attention.qkv_proj.bias"]).split(w, -1)
        q, k = G.rotate(q.view(B, S, H, 64), cos, sin), G.rotate(k.view(B, S, H, 64), cos, sin)
        o = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.view(B, S, H, 64).transpose(1, 2),
                                           attn_mask=keep)
        o = F.linear(o.transpose(1, 2).reshape(B, S, w), sd[p + "attention.o_proj.weight"], sd[p + "attention.o_proj.bias"])
        x = F.layer_norm(x + o, (w,), sd[p + "attn_ln.weight"], sd[p + "attn_ln.bias"], cfg.ln_eps)
        up, gate = F.linear(x, sd[p + "mlp.up_gate_proj.weight"]).split(cfg.mlp, -1)
        d = F.linear(F.gelu(gate) * up, sd[p + "mlp.down_proj.weight"], sd[p + "mlp.down_proj.bias"])
        x = F.layer_norm(x + d, (w,), sd[p + "mlp_ln.weight"], sd[p + "mlp_ln.bias"], cfg.ln_eps)
    m = mask[..., None].to(x.dtype)
    return F.normalize((x * m).sum(1) / m.sum(1), dim=1)


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in q.split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def _time(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/gte_probe.py measures on a GPU; none is visible")
    torch.backends.cuda.matmul.allow_tf32 = False
    res = {"card": _card(), "model": G.NAME, "steps": args.steps, "warmup": args.warmup, "shapes": {}}
    cfg = G.STELLA
    sd = G.make_gte_weights(cfg, seed=1234)
    enc = Encoder("gte", G.engine_config(cfg), sd, max_batch=256)
    tsd = {k: v.cuda() for k, v in sd.items()}
    del sd
    out = torch.empty(256, cfg.width, dtype=torch.float32, device="cuda")
    inputs = {}
    for name, B, S in SHAPES:
        lens = torch.randint(S // 2, S + 1, (B,), generator=torch.Generator().manual_seed(B + S))
        lens[0] = S
        ids, mask = G.ragged_ids(torch.Generator().manual_seed(S), lens.tolist(), S, cfg.vocab)
        inputs[name] = (ids.cuda(), mask.cuda(), ids.int().cuda(), mask.int().cuda())
    for name, B, S in SHAPES:
        ids, mask, ids32, mask32 = inputs[name]
        th = G.rope_angles(cfg, S).cuda()
        cos, sin = th.cos().float(), th.sin().float()

        def engine():
            enc.encode_tokens_device(ids32.data_ptr(), mask32.data_ptr(), B, S, out.data_ptr(), sync=True)

        def reference():
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                return torch_forward(tsd, cfg, ids, mask, cos, sin)

        eng, ref = [], []
        for _ in range(3):   # alternated
            eng.append(_time(engine, args.steps, args.warmup))
            ref.append(_time(reference, args.steps, args.warmup))
        cos_min = float(F.cosine_similarity(out[:B].double(), reference().double(), dim=1).min())
        res["shapes"][name] = {"B": B, "S": S, "engine_ms": float(np.median(eng)), "torch_bf16_sdpa_ms":
                               float(np.median(ref)), "engine_rounds_ms": eng, "torch_rounds_ms": ref,
                               "min_cosine_vs_torch_bf16": cos_min}
        print(json.dumps({name: res["shapes"][name]}), flush=True)
    # b200_model_profile: GEMM and attention device time of one b64 x 512 forward, against its whole device time
    ids, mask, ids32, mask32 = inputs["b64x512"]
    enc.set_profiling(True)
    enc.encode_tokens_device(ids32.data_ptr(), mask32.data_ptr(), 64, 512, out.data_ptr(), sync=True)
    prof = enc.profile()
    enc.set_profiling(False)
    enc.encode_tokens_device(ids32.data_ptr(), mask32.data_ptr(), 64, 512, out.data_ptr(), sync=True)
    total_ms = enc.last_timing()[0]
    other = total_ms - prof["gemm_ms"] - prof["attention_ms"]
    res["b64x512_profile"] = {**prof, "forward_ms": total_ms, "other_ms": other, "other_share": other / total_ms}
    # which kernels make up the rest
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as p:
        enc.encode_tokens_device(ids32.data_ptr(), mask32.data_ptr(), 64, 512, out.data_ptr(), sync=True)
        torch.cuda.synchronize()
    cls_us = {}
    for e in p.key_averages():
        t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        if e.key.startswith(("Memcpy", "Memset")) or t <= 0:
            continue
        cls = next((c for c in ("rope_qk", "geglu", "layernorm", "embed_ln", "bert_head", "attention", "gemm")
                    if c in e.key), "other")
        cls_us[cls] = cls_us.get(cls, 0.0) + t
    total = sum(cls_us.values())
    res["b64x512_kernel_share"] = {c: us / total for c, us in sorted(cls_us.items())}
    res["b64x512_rope_geglu_share"] = (cls_us.get("rope_qk", 0.0) + cls_us.get("geglu", 0.0)) / total
    enc.close()
    print(json.dumps({k: res[k] for k in ("card", "b64x512_profile", "b64x512_kernel_share",
                                          "b64x512_rope_geglu_share")}), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
