"""Dev probe for the 384-wide BERT embedders (head_dim 32), not a bench line.  Needs a GPU; prints JSON lines.

  1. attention kernel alone (debug_attention_time, key-length mask, every key valid) vs
     torch.nn.functional.scaled_dot_product_attention in bf16 on q / k / v already split into [B, H, S, 32];
  2. device-resident forward (ids on the device, mean pooling + L2 normalise, seeded weights) vs HF BertModel built
     from the same config, in fp32 (what the reference runs on CUDA) and in bf16, both with transformers' SDPA attention.
Times are host clocks around `iters` calls that end in a device synchronise, after `warmup` calls of the same shape.

    python tools/small_bert_probe.py [iters]
"""
import json
import subprocess
import sys
import time

import torch

sys.path.insert(0, ".")
from marqo_b200 import _native as N, model_registry as R, weights as Wt  # noqa: E402
from marqo_b200.engine import Encoder, debug_attention_time  # noqa: E402

ITERS = int(sys.argv[1]) if len(sys.argv) > 1 else 50
WARMUP = 5


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in q.split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def _wall(fn, iters):
    for _ in range(WARMUP):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / iters * 1e3


def attention(B, S, H=12, hd=32):
    W = H * hd
    ms = debug_attention_time(B, S, W, H, mask=2, iters=ITERS)
    q, k, v = (torch.randn(B, H, S, hd, device="cuda", dtype=torch.bfloat16) for _ in range(3))
    sdpa = _wall(lambda: torch.nn.functional.scaled_dot_product_attention(q, k, v), ITERS)
    flops = 4.0 * B * H * S * S * hd
    return {"probe": "attention", "B": B, "S": S, "H": H, "head_dim": hd, "engine_us": ms * 1e3,
            "sdpa_bf16_us": sdpa * 1e3, "engine_TFLOPs": flops / ms / 1e9, "speedup_vs_sdpa": sdpa / ms}


def forward(name, B, S):
    from transformers import BertConfig, BertModel
    arch = R.get_model_properties(name)["arch"]
    sd = Wt.random_bert_weights(arch, 1234)
    enc = Encoder("bert", arch, sd, max_batch=B)
    g = torch.Generator(device="cuda").manual_seed(0)
    ids = torch.randint(1000, 30000, (B, S), dtype=torch.int32, device="cuda", generator=g)
    out = torch.empty(B, arch["width"], dtype=torch.float32, device="cuda")
    engine = _wall(lambda: enc.encode_tokens_device(ids.data_ptr(), None, B, S, out.data_ptr()), ITERS)
    hc = BertConfig(vocab_size=arch["vocab"], hidden_size=arch["width"], num_hidden_layers=arch["layers"],
                    num_attention_heads=arch["heads"], intermediate_size=arch["mlp"],
                    max_position_embeddings=arch["max_pos"], type_vocab_size=arch["type_vocab"], hidden_act="gelu",
                    attn_implementation="sdpa")
    model = BertModel(hc, add_pooling_layer=False).cuda().eval()
    model.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=False)
    ids64, mask = ids.long(), torch.ones(B, S, dtype=torch.long, device="cuda")

    def hf():
        with torch.no_grad():
            last = model(input_ids=ids64, attention_mask=mask).last_hidden_state
            emb = (last * mask[..., None]).sum(1) / mask.sum(1, keepdim=True)
            return torch.nn.functional.normalize(emb.float(), dim=-1)

    ref32 = hf()
    fp32 = _wall(hf, ITERS)
    model = model.to(torch.bfloat16)
    bf16 = _wall(hf, ITERS)
    cos = float(torch.nn.functional.cosine_similarity(out.double(), ref32.double(), dim=-1).min())
    enc.close()
    return {"probe": "forward", "model": name, "B": B, "S": S, "engine_ms": engine, "hf_fp32_ms": fp32,
            "hf_bf16_sdpa_ms": bf16, "engine_items_per_s": B / engine * 1e3, "hf_fp32_items_per_s": B / fp32 * 1e3,
            "hf_bf16_items_per_s": B / bf16 * 1e3, "min_cos_vs_hf_fp32": cos}


def main():
    if not torch.cuda.is_available() or N.device_count() < 1:
        sys.exit("small_bert_probe: needs an sm_90 GPU")
    torch.backends.cuda.matmul.allow_tf32 = False
    print(json.dumps(_card()), flush=True)
    for B, S in ((1, 16), (256, 128), (64, 512)):
        print(json.dumps(attention(B, S)), flush=True)
    for name, B, S in (("hf/all-MiniLM-L6-v2", 256, 128), ("hf/all-MiniLM-L6-v2", 1, 16), ("hf/e5-small-v2", 64, 512)):
        print(json.dumps(forward(name, B, S)), flush=True)


if __name__ == "__main__":
    main()
