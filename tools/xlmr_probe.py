"""Dev probe for the multilingual-e5 embedders (XLM-R), not a bench line.  Prints JSON lines.

  1. host (CPU) tokenizer throughput: texts/s of the C++ SentencePiece Unigram tokenizer on the test fixture model
     (tests/golden/unigram_golden.model) beside the C++ WordPiece tokenizer, both over the same multilingual texts;
  2. with a GPU: device-resident forward of hf/multilingual-e5-large (XLM-R) and hf/e5-large-v2 (BERT) at b64 x 512,
     seeded weights, alternated `rounds` times in one process.  The two share every layer shape (width 1024, 24 layers,
     16 heads, mlp 4096); only the embedding step and the word table (250002 vs 30522 rows) differ.
Times are CUDA events around `iters` calls after `warmup` calls of the same shape; the card's name, power limit and
SM clock limit are read in the same run.

    python tools/xlmr_probe.py [iters] [rounds]
"""
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, ".")
from marqo_b200 import model_registry as R, weights as Wt  # noqa: E402
from marqo_b200.tokenizers import WordPieceTokenizer, XLMRTokenizer  # noqa: E402

ITERS = int(sys.argv[1]) if len(sys.argv) > 1 else 20
ROUNDS = int(sys.argv[2]) if len(sys.argv) > 2 else 3
WARMUP = 3
FIXTURE = Path(__file__).resolve().parent.parent / "tests" / "golden" / "unigram_golden.model"


def tokenizers():
    rng = np.random.default_rng(0)
    alphabets = ["abcdefghijklmnopqrstuvwxyz", "абвгдежзийклмнопрстуфхцчшщыэюя", "東京大学日本語中文字学生先生",
                 "aeiouéèêàçñüöäß"]
    words = ["".join(rng.choice(list(a)) for _ in range(int(rng.integers(1, 8)))) for a in alphabets for _ in range(1000)]
    texts = [" ".join(words[int(i)] for i in rng.integers(0, len(words), size=int(rng.integers(5, 120))))
             for _ in range(20000)]
    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + sorted(set(words))[:3000]

    def rate(tok):
        best = 1e9
        for _ in range(3):
            t0 = time.perf_counter()
            tok(texts, max_length=512)
            best = min(best, time.perf_counter() - t0)
        return len(texts) / best

    return {"probe": "tokenizer_cpu", "texts": len(texts), "mean_words": float(np.mean([len(t.split()) for t in texts])),
            "unigram_fixture_texts_per_s": rate(XLMRTokenizer(str(FIXTURE))),
            "wordpiece_texts_per_s": rate(WordPieceTokenizer(("\n".join(vocab) + "\n").encode()))}


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in q.split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def forward(B=64, S=512):
    import torch
    from marqo_b200.engine import Encoder
    encs, ids = {}, {}
    for name in ("hf/multilingual-e5-large", "hf/e5-large-v2"):
        arch = R.get_model_properties(name)["arch"]
        kind = arch.get("kind", "bert")
        sd = Wt.random_xlmr_weights(arch, 1234) if kind == "xlmr" else Wt.random_bert_weights(arch, 1234)
        encs[name] = Encoder(kind, arch, sd, max_batch=B)
        del sd
        g = torch.Generator(device="cuda").manual_seed(0)
        ids[name] = torch.randint(4, arch["vocab"], (B, S), dtype=torch.int32, device="cuda", generator=g)
    out = torch.empty(B, 1024, dtype=torch.float32, device="cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(name):
        enc, x = encs[name], ids[name]
        run = lambda: enc.encode_tokens_device(x.data_ptr(), None, B, S, out.data_ptr(), sync=False)  # noqa: E731
        for _ in range(WARMUP):
            run()
        torch.cuda.synchronize()
        e0.record(torch.cuda.current_stream())
        for _ in range(ITERS):
            run()
        # the engine runs on its own stream: synchronise the device before the closing event
        torch.cuda.synchronize()
        e1.record(torch.cuda.current_stream())
        e1.synchronize()
        return e0.elapsed_time(e1) / ITERS

    rows = {n: [] for n in encs}
    for _ in range(ROUNDS):
        for n in encs:
            rows[n].append(timed(n))
    res = {"probe": "forward", "B": B, "S": S, "iters": ITERS, "rounds": ROUNDS}
    for n, ms in rows.items():
        res[n] = {"ms_per_call": ms, "median_ms": float(np.median(ms)), "items_per_s": B / float(np.median(ms)) * 1e3}
    res["xlmr_over_bert"] = res["hf/multilingual-e5-large"]["median_ms"] / res["hf/e5-large-v2"]["median_ms"]
    for e in encs.values():
        e.close()
    return res


def main():
    print(json.dumps(tokenizers()), flush=True)
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if not has_gpu:
        print(json.dumps({"probe": "forward", "skipped": "no GPU"}), flush=True)
        return
    print(json.dumps(_card()), flush=True)
    print(json.dumps(forward()), flush=True)


if __name__ == "__main__":
    main()
