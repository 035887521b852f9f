"""Reranking on one GPU: B200CrossEncoder.predict against torch fp32 transformers.BertForSequenceClassification on the
same card, same seeded weights (no downloads), at the two sizes a reranked search meets:

  1. latency: one rerank request, 10 hits x 5 chunks = 50 (query, chunk) pairs of at most 128 tokens, predict's
     default batch_size 32 (two batches), ms per request;
  2. throughput: 1024 pairs of 256 tokens in batches of 256, pairs/s.

The torch side runs what CrossEncoder.predict runs per batch: the same tokenizer output as int64 tensors on the GPU,
the model's forward under no_grad, the sigmoid, and the copy back.  Medians over --steps calls after --warmup; the
largest |score difference| between the two is printed beside each time.  Also prints the card's name and power limit,
read in the same process.

    python tools/rerank_probe.py [--models tinybert-l2,minilm-l6,minilm-l12] [--steps 20] [--warmup 3] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from marqo_b200 import model_registry as R  # noqa: E402
from marqo_b200.cross_encoder import B200CrossEncoder  # noqa: E402
from marqo_b200.weights import random_cross_encoder_weights  # noqa: E402

NAMES = {"tinybert-l2": "cross-encoder/ms-marco-TinyBERT-L-2", "minilm-l6": "cross-encoder/ms-marco-MiniLM-L-6-v2",
         "minilm-l12": "cross-encoder/ms-marco-MiniLM-L-12-v2"}
# a vocabulary of 2000 distinct whole words: every word is one WordPiece, so a text of k words is k tokens
WORDS = [f"w{i}" for i in range(2000)]


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
    return float(np.median(ts))


def pairs(rng, n, q_words, p_words):
    text = lambda k: " ".join(rng.choice(WORDS, k))
    return [[text(int(rng.integers(3, q_words + 1))), text(int(rng.integers(p_words // 2, p_words + 1)))]
            for _ in range(n)]


def torch_model(arch, sd):
    import transformers
    cfg = transformers.BertConfig(vocab_size=arch["vocab"], hidden_size=arch["width"],
                                  num_hidden_layers=arch["layers"], num_attention_heads=arch["heads"],
                                  intermediate_size=arch["mlp"], max_position_embeddings=arch["max_pos"],
                                  type_vocab_size=arch["type_vocab"], num_labels=arch["num_labels"],
                                  layer_norm_eps=1e-12, attn_implementation="eager")
    m = transformers.BertForSequenceClassification(cfg)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=False)
    return m.eval().cuda()


def torch_predict(model, tokenizer, ps, batch_size, max_length):
    out = []
    with torch.no_grad():
        for o in range(0, len(ps), batch_size):
            part = ps[o:o + batch_size]
            tok = tokenizer([a.strip() for a, _ in part], [b.strip() for _, b in part], padding=True,
                            truncation="longest_first", max_length=max_length)
            feats = {k: torch.from_numpy(v).cuda() for k, v in tok.items()}
            out.append(torch.sigmoid(model(**feats).logits)[:, 0].cpu())
    return torch.cat(out).numpy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="tinybert-l2,minilm-l6,minilm-l12")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False   # torch's model in fp32, as the reranker runs it
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    result = {"gpu": smi, "torch_tf32": False, "models": {}}
    print("GPU:", smi)
    vocab_dir = tempfile.mkdtemp()
    vocab = os.path.join(vocab_dir, "vocab.txt")
    with open(vocab, "w") as f:
        f.write("\n".join(["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + WORDS) + "\n")
    rng = np.random.default_rng(0)
    cases = {"latency_50x128": (pairs(rng, 50, 12, 120), 32, 128),
             "throughput_1024x256": (pairs(rng, 1024, 20, 240), 256, 256)}
    for key in args.models.split(","):
        name = NAMES[key]
        arch = R.CROSS_ENCODER_MODELS[name]["arch"]
        sd = random_cross_encoder_weights(arch, 7)
        mine = B200CrossEncoder(name, max_length=512, device="cuda", default_activation_function=torch.nn.Sigmoid(),
                                weights=sd, vocab_file=vocab)
        ref = torch_model(arch, sd)
        row = {}
        for case, (ps, bs, max_length) in cases.items():
            mine.max_length = max_length
            got = mine.predict(ps, batch_size=bs)
            exp = torch_predict(ref, mine.tokenizer, ps, bs, max_length)
            t_mine = timed(lambda: mine.predict(ps, batch_size=bs), args.steps, args.warmup)
            t_ref = timed(lambda: torch_predict(ref, mine.tokenizer, ps, bs, max_length), args.steps, args.warmup)
            row[case] = {"pairs": len(ps), "batch_size": bs, "max_length": max_length, "b200_ms": 1e3 * t_mine,
                         "torch_fp32_ms": 1e3 * t_ref, "speedup": t_ref / t_mine,
                         "b200_pairs_per_s": len(ps) / t_mine, "torch_pairs_per_s": len(ps) / t_ref,
                         "max_abs_score_diff": float(np.abs(got - exp).max())}
            print(f"{key:12s} {case:20s} b200 {1e3 * t_mine:8.2f} ms  torch fp32 {1e3 * t_ref:8.2f} ms  "
                  f"x{t_ref / t_mine:6.2f}  max|diff| {row[case]['max_abs_score_diff']:.2e}", flush=True)
        result["models"][name] = row
        mine.close()
        del ref
        torch.cuda.empty_cache()
    print(json.dumps(result))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
