"""MPNet (hf/all-mpnet-base-v1/v2, hf/all_datasets_v3/v4_mpnet-base) on the host: the registry entries vs the
reference's, the relative-position buckets the runtime builds its bias table from vs transformers, the CPU oracle
(tests/_mpnet_oracle.py) vs transformers.MPNetModel and vs the reference's HuggingFaceModel.encode
(tests/golden/mpnet_golden.npz), and the C++ MPNet tokenizer vs transformers.MPNetTokenizer."""
import json
import random
from pathlib import Path

import numpy as np
import pytest
import torch

import _mpnet_oracle as M
from marqo_b200 import model_registry as R

GOLDEN_DIR = Path(__file__).resolve().parent / "golden"
MPNET_NAMES = ("hf/all-mpnet-base-v1", "hf/all-mpnet-base-v2", "hf/all_datasets_v3_mpnet-base",
               "hf/all_datasets_v4_mpnet-base")


def test_mpnet_entries_are_the_reference_entries():
    ref = json.loads((GOLDEN_DIR / "hf_registry_golden.json").read_text())
    assert sorted(R.MPNET_MODELS) == sorted(MPNET_NAMES)
    for name in MPNET_NAMES:
        entry = R.MPNET_MODELS[name]
        assert {k: v for k, v in entry.items() if k != "arch"} == dict(ref[name], type=R.TYPE_HF), name
        assert R.get_model_properties(name) == entry
        assert R.find_model(name) is entry and R.all_models()[name] is entry
        a = entry["arch"]
        assert a["kind"] == "mpnet" and a["width"] == entry["dimensions"] and a["width"] // a["heads"] == 64
        assert (a["vocab"], a["max_pos"], a["pad_id"], a["ln_eps"], a["rel_buckets"], a["rel_max_distance"]) == \
            (30527, 514, 1, 1e-5, 32, 128)
    assert not set(R.MPNET_MODELS) & set(R.MODELS)


def test_validate_model_properties_finds_mpnet_by_name():
    from marqo_b200 import s2_inference as s2
    props = s2.validate_model_properties("hf/all-mpnet-base-v2", None)
    assert props["arch"]["kind"] == "mpnet"
    custom = s2.validate_model_properties("my-mpnet", {"name": "sentence-transformers/all-mpnet-base-v2",
                                                       "dimensions": 768, "type": "hf"})
    assert custom["arch"] == R.MPNET_MODELS["hf/all-mpnet-base-v2"]["arch"]


def test_bucket_table_matches_transformers(native_lib):
    """The buckets the runtime's bias table uses, for every key - query distance |d| <= 1023."""
    from transformers.models.mpnet.modeling_mpnet import MPNetEncoder
    from marqo_b200.engine import relative_position_buckets
    n = 1024
    rel = torch.arange(-(n - 1), n)
    want = MPNetEncoder.relative_position_bucket(rel, num_buckets=32, max_distance=128).numpy()
    np.testing.assert_array_equal(relative_position_buckets(n), want)
    np.testing.assert_array_equal(M.relative_position_bucket(rel).numpy(), want)
    # the table in the issue text: |n| 8-11 -> 8, 12-15 -> 9, ..., >= 91 -> 15; +16 for keys after the query
    for lo, hi, b in ((8, 11, 8), (12, 15, 9), (16, 22, 10), (23, 31, 11), (32, 45, 12), (46, 63, 13), (64, 90, 14),
                      (91, 1023, 15)):
        for d in (lo, hi):
            assert want[n - 1 - d] == b and want[n - 1 + d] == b + 16


def _hf_model(cfg, sd):
    from transformers import MPNetModel
    m = MPNetModel(M.hf_config(cfg), add_pooling_layer=False).eval()
    res = m.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys and all("position_ids" in k for k in res.missing_keys)
    return m


def _hf_mean_pool(m, ids, mask):
    with torch.no_grad():
        last = m(input_ids=ids, attention_mask=mask).last_hidden_state
    last = last.masked_fill(~mask[..., None].bool(), 0.0)
    return torch.nn.functional.normalize(last.sum(dim=1) / mask.sum(dim=1)[..., None], p=2, dim=1)


@pytest.mark.parametrize("cfg", [M.tiny_mpnet(), M.MpnetCfg(256, 2, 4, 1024, vocab=3000, max_pos=202)],
                         ids=["tiny", "hd64"])
def test_oracle_matches_transformers(cfg):
    """mpnet_encode vs MPNetModel (eager, dropout 0) on ragged masks and on rows holding the pad id mid-sequence."""
    sd = M.make_mpnet_weights(cfg, seed=21)
    m = _hf_model(cfg, sd)
    S = cfg.max_pos - cfg.pad_id - 1
    g = torch.Generator().manual_seed(4)
    ids = torch.randint(5, cfg.vocab, (5, S), generator=g)
    ids[:, 0] = 0
    mask = torch.ones(5, S, dtype=torch.long)
    for b, L in enumerate([S, 12, 1, 27, S - 3]):
        ids[b, L - 1] = 2
        mask[b, L:] = 0
        ids[b, L:] = cfg.pad_id
    ids[3, 5] = cfg.pad_id            # an id 1 inside the text: its position is the pad's, later ones shift down
    ids[0, S // 2] = cfg.pad_id
    torch.testing.assert_close(M.mpnet_encode(sd, cfg, ids, mask), _hf_mean_pool(m, ids, mask), rtol=1e-4, atol=1e-4)


def test_oracle_matches_reference_golden():
    """The oracle vs the reference's own HuggingFaceModel.encode (tests/golden/make_mpnet_golden.py)."""
    z = np.load(GOLDEN_DIR / "mpnet_golden.npz")
    cfg = M.tiny_mpnet()
    sd = M.make_mpnet_weights(cfg, seed=int(z["seed"]))
    ids, mask = torch.from_numpy(z["ids"]), torch.from_numpy(z["mask"])
    np.testing.assert_allclose(M.mpnet_encode(sd, cfg, ids, mask).numpy(), z["vec"], rtol=0, atol=2e-5)
    np.testing.assert_allclose(M.mpnet_encode(sd, cfg, ids, mask, normalize=False).numpy(), z["vec_unnormalized"],
                               rtol=1e-4, atol=1e-4)


# ------------------------------------------------------------------------------------------------ tokenizer
@pytest.fixture(scope="module")
def vocab_file(tmp_path_factory):
    f = tmp_path_factory.mktemp("mpnet_vocab") / "vocab.txt"
    f.write_text("\n".join(M.synthetic_vocab(1000)) + "\n")
    return f


@pytest.fixture(scope="module")
def tokenizers(vocab_file, native_lib):
    from transformers import MPNetTokenizer as HF
    from marqo_b200.tokenizers import MPNetTokenizer
    return HF(str(vocab_file)), MPNetTokenizer(vocab_file)


def _same(tokenizers, sentences, max_length):
    hf, ours = tokenizers
    want = hf(sentences, padding=True, truncation=True, max_length=max_length, return_tensors="np")
    got = ours(sentences, padding=True, truncation=True, max_length=max_length, return_tensors="np")
    assert set(got) == {"input_ids", "attention_mask"}
    np.testing.assert_array_equal(got["input_ids"], want["input_ids"])
    np.testing.assert_array_equal(got["attention_mask"], want["attention_mask"])


HAND_PICKED = [
    "the cat sat on the mat", "<s>", "</s>", "<pad>", "<mask>", " <mask>x", "hello<mask>world", "[UNK]", "[CLS]",
    "[SEP] [MASK]", "<unk>", "<s> the cat </s> <pad> sat", "Hello, World!  UNABLE playing", "ÀÉÎ õü çat",
    "x" * 120, "un##able", "<mask><mask> <s></s>", "[cls]the[sep]", "", "   ", "a\tb\nc", "日本 the 中文",
]


def test_tokenizer_hand_picked(tokenizers):
    _same(tokenizers, HAND_PICKED, 128)
    for s in HAND_PICKED:
        _same(tokenizers, [s], 128)


@pytest.mark.parametrize("max_length", [2, 3, 8, 128])
def test_tokenizer_truncation_and_padding(tokenizers, max_length):
    _same(tokenizers, ["the cat sat on the mat and ran", "hello", "<mask> the cat " * 20, "", "playing unable w12 w7"],
          max_length)


def test_tokenizer_random_sentences(tokenizers):
    rng = random.Random(5)
    words = M.synthetic_vocab(1000)[9:400] + ["<s>", "</s>", "<pad>", "<mask>", "[UNK]", "[CLS]", "<unk>", "Hello,",
                                              "UNABLE", "x!y", "zzz", "ñ"]
    sentences = [" ".join(rng.choice(words) for _ in range(rng.randint(0, 40))) for _ in range(300)]
    for i in range(0, 300, 50):
        _same(tokenizers, sentences[i:i + 50], 64)
