"""Generate tests/golden/mpnet_golden.npz by RUNNING THE REFERENCE'S OWN CODE in the build container (/root/reference
is mounted there and nowhere else; the GPU box only sees the committed fixture).

What is executed from /root/reference (via the import shim in _reference_import.py):
  * marqo.core.inference.embedding_models.hugging_face_model.HuggingFaceModel.encode on a config-instantiated
    transformers MPNetModel carrying the MPNet oracle's seeded weights (tests/_mpnet_oracle.py, tiny_mpnet), with a
    transformers MPNetTokenizer on a synthetic vocabulary — the (a5) recipe of make_reference_golden.py.

Caveat recorded in the fixture: transformers here is 5.5.0 (the reference pins 4.41.2), torch 2.11 (pins 1.12.1).

Run:  python tests/golden/make_mpnet_golden.py
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import _reference_import as RI  # noqa: E402

RI.install()
import torch  # noqa: E402
import transformers  # noqa: E402

import _mpnet_oracle as M  # noqa: E402
from marqo.core.inference.embedding_models.hugging_face_model import HuggingFaceModel  # noqa: E402
from transformers import MPNetModel, MPNetTokenizer  # noqa: E402

SEED = 2024
cfg = M.tiny_mpnet()
sd = M.make_mpnet_weights(cfg, seed=SEED)
model = MPNetModel(M.hf_config(cfg), add_pooling_layer=False).eval()
model.load_state_dict(sd, strict=False)
with tempfile.TemporaryDirectory() as td:
    vf = os.path.join(td, "vocab.txt")
    with open(vf, "w") as f:
        f.write("\n".join(M.synthetic_vocab(cfg.vocab)) + "\n")
    tok = MPNetTokenizer(vf, do_lower_case=True)
ref_model = HuggingFaceModel.__new__(HuggingFaceModel)   # bypass load(): no network, no checkpoint
ref_model.device = "cpu"
ref_model._model = model
ref_model._tokenizer = tok
ref_model.model_properties = type("P", (), {"tokens": 48, "pooling_method": "mean"})()
ref_model._pooling_func = HuggingFaceModel._average_pool_func
rng = np.random.default_rng(7)
words = M.synthetic_vocab(cfg.vocab)[9:-1]
sentences = [" ".join(words[int(x)] for x in rng.integers(0, len(words), size=n)) for n in (3, 30, 11, 1, 60, 17)]
sentences[2] += " <pad> the <mask> cat"            # a pad id inside the text
vec = ref_model.encode(sentences, normalize=True)
vec_un = ref_model.encode(sentences, normalize=False)
enc = tok(sentences, padding=True, truncation=True, max_length=48, return_tensors="np")
np.savez_compressed(
    os.path.join(HERE, "mpnet_golden.npz"),
    ids=enc["input_ids"].astype(np.int32), mask=enc["attention_mask"].astype(np.int32),
    vec=np.asarray(vec, dtype=np.float32), vec_unnormalized=np.asarray(vec_un, dtype=np.float32),
    seed=np.int64(SEED),
    meta=np.asarray(f"HuggingFaceModel.encode (mean pooling, tokens 48) on MPNetModel(tiny_mpnet) with "
                    f"_mpnet_oracle.make_mpnet_weights(seed={SEED}); transformers {transformers.__version__} "
                    f"(reference pins 4.41.2), torch {torch.__version__} (reference pins 1.12.1)"))
print("wrote", os.path.join(HERE, "mpnet_golden.npz"), enc["input_ids"].shape)
