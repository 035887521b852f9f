"""The text reranker's cross-encoders on the CPU: WordPiece pair encoding against HF tokenizers' BERT WordPiece
pipeline, the one BertTokenizerFast runs (ids, token types and mask under longest_first truncation), the cross-encoder oracle against transformers'
BertForSequenceClassification, the CROSS_ENCODER_MODELS table, and the CrossEncoder factory's routing."""
import random

import numpy as np
import pytest
import torch

import _cross_encoder_oracle as O

WORDS = ["the", "quick", "brown", "fox", "jump", "over", "lazy", "dog", "hello", "world", "search", "vector", "marqo",
         "is", "a", "re", "rank", "query", "passage", "un", "able", "token", "cafe"]
VOCAB = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + WORDS + ["##s", "##ing", "##ed", "##er", "##able", "##ly"] + \
        list("!,.?'-") + list("0123456789")


@pytest.fixture(scope="module")
def pair_tokenizers(native_lib, tmp_path_factory):
    from marqo_b200.tokenizers import WordPieceTokenizer
    from oracle import tokenizers as OT
    path = tmp_path_factory.mktemp("vocab") / "vocab.txt"
    path.write_text("\n".join(VOCAB) + "\n", encoding="utf-8")
    return WordPieceTokenizer(str(path)), OT.bert_wordpiece(VOCAB)


def _hf_pairs(tok, a, b, max_length):
    tok.enable_truncation(max_length=max_length, strategy="longest_first")
    tok.enable_padding(pad_id=tok.token_to_id("[PAD]"), pad_token="[PAD]")
    enc = tok.encode_batch(list(zip(a, b)))
    return {k: np.asarray([getattr(e, attr) for e in enc], dtype=np.int64)
            for k, attr in (("input_ids", "ids"), ("token_type_ids", "type_ids"), ("attention_mask", "attention_mask"))}


def _words(n, rng):
    return " ".join(rng.choice(WORDS) for _ in range(n))


def _same_pairs(pair_tokenizers, a, b, max_length):
    mine, hf = pair_tokenizers
    got = mine(list(a), list(b), padding=True, truncation="longest_first", max_length=max_length)
    ref = _hf_pairs(hf, a, b, max_length)
    for k in ("input_ids", "token_type_ids", "attention_mask"):
        np.testing.assert_array_equal(got[k], ref[k], err_msg=k)
    return got


# (len a, len b, max_length): the budget m = max_length - 3 ids for the two texts
@pytest.mark.parametrize("la,lb,max_length", [
    (3, 4, 16),     # both fit
    (20, 3, 16),    # only A over the budget
    (3, 20, 16),    # only B over
    (20, 25, 16),   # both over, even budget (13 -> 6 + 7)
    (20, 25, 14),   # both over, odd budget
    (9, 9, 12),     # equal lengths over the budget
    (15, 30, 12),   # n1 > m: the shorter side alone is over the budget
    (0, 12, 8),     # an empty side
    (12, 0, 8),
    (5, 5, 3),      # budget 0: "[CLS] [SEP] [SEP]"
])
def test_pair_truncation_cases(pair_tokenizers, la, lb, max_length):
    rng = random.Random(la * 100 + lb)
    got = _same_pairs(pair_tokenizers, [_words(la, rng)], [_words(lb, rng)], max_length)
    assert got["input_ids"].shape[1] <= max_length


def test_pair_batch_random(pair_tokenizers):
    rng = random.Random(7)
    for max_length in (8, 17, 64, 512):
        a = [_words(rng.randrange(0, 40), rng) + rng.choice(["", "!", " 12 cafe's"]) for _ in range(24)]
        b = [_words(rng.randrange(0, 60), rng) for _ in range(24)]
        _same_pairs(pair_tokenizers, a, b, max_length)


def test_pair_strip_matches_predict(pair_tokenizers):
    """predict strips each text first; stripped or not, BERT's pre-tokenizer drops the outer whitespace."""
    a, b = ["  hello world \n", "\tthe fox "], [" a re rank query\t\t", "passage  "]
    got = _same_pairs(pair_tokenizers, [x.strip() for x in a], [y.strip() for y in b], 32)
    raw = _same_pairs(pair_tokenizers, a, b, 32)
    np.testing.assert_array_equal(got["input_ids"], raw["input_ids"])


def test_pair_call_refusals(pair_tokenizers):
    mine, _ = pair_tokenizers
    with pytest.raises(ValueError):
        mine(["a"], ["b"], padding=True, truncation=True, max_length=16)
    with pytest.raises(ValueError):
        mine(["a"], ["b", "c"], padding=True, truncation="longest_first", max_length=16)
    single = mine(["hello world"], padding=True, truncation=True, max_length=16)   # the single-text call is unchanged
    assert not single["token_type_ids"].any()


@pytest.mark.parametrize("name", ["cross-encoder/ms-marco-TinyBERT-L-2", "cross-encoder/ms-marco-MiniLM-L-6-v2"])
def test_oracle_matches_transformers(name):
    a = O.arch(name, layers=2, vocab=500)
    sd = O.weights(a, seed=11)
    rng = np.random.default_rng(0)
    n, S = 5, 40
    lens = np.array([40, 3, 17, 29, 8])
    ids = rng.integers(5, 500, size=(n, S))
    mask = (np.arange(S)[None] < lens[:, None]).astype(np.int64)
    types = ((np.arange(S)[None] > lens[:, None] // 2) & (mask == 1)).astype(np.int64)
    ids[mask == 0] = 0
    pooled, logits = O.forward(sd, a, ids, mask, types)
    hp, hl = O.hf_forward(sd, a, ids, mask, types)
    torch.testing.assert_close(pooled, hp, rtol=0, atol=2e-5)
    torch.testing.assert_close(logits, hl, rtol=0, atol=2e-5)
    assert logits.shape == (n, 1)


TABLE = {
    "cross-encoder/ms-marco-TinyBERT-L-2": (128, 2, 2, 512), "cross-encoder/ms-marco-TinyBERT-L-2-v2": (128, 2, 2, 512),
    "cross-encoder/ms-marco-MiniLM-L-2-v2": (384, 2, 12, 1536), "cross-encoder/ms-marco-MiniLM-L-4-v2": (384, 4, 12, 1536),
    "cross-encoder/ms-marco-MiniLM-L-6-v2": (384, 6, 12, 1536),
    "cross-encoder/ms-marco-MiniLM-L-12-v2": (384, 12, 12, 1536),
}


def test_cross_encoder_table():
    from marqo_b200 import model_registry as R
    assert set(R.CROSS_ENCODER_MODELS) == set(TABLE)
    for name, (w, layers, heads, mlp) in TABLE.items():
        a = R.CROSS_ENCODER_MODELS[name]["arch"]
        assert (a["width"], a["layers"], a["heads"], a["mlp"]) == (w, layers, heads, mlp)
        assert (a["vocab"], a["max_pos"], a["type_vocab"], a["num_labels"]) == (30522, 512, 2, 1)
        assert R.find_model(name) is None and name not in R.served_models() and name not in R.all_models()


class _Stand:
    def __init__(self, model_name, *args, **kwargs):
        self.model_name, self.args, self.kwargs = model_name, args, kwargs


class _Original(_Stand):
    pass


class _Served(_Stand):
    pass


def test_factory_routes_served_names():
    from marqo_b200.cross_encoder import make_cross_encoder_factory
    f = make_cross_encoder_factory(_Original, served=_Served)
    act = torch.nn.Sigmoid()
    m = f("cross-encoder/ms-marco-MiniLM-L-6-v2", max_length=512, device="cuda", default_activation_function=act)
    assert isinstance(m, _Served)
    assert m.kwargs == {"max_length": 512, "device": "cuda", "default_activation_function": act}
    m = f("cross-encoder/ms-marco-TinyBERT-L-2", None, 256, "cuda:1")   # CrossEncoder's positional order
    assert isinstance(m, _Served) and m.kwargs == {"max_length": 256, "device": "cuda:1"}
    for name, device in (("cross-encoder/ms-marco-electra-base", "cuda"), ("cross-encoder/ms-marco-TinyBERT-L-4", "cuda"),
                         ("cross-encoder/ms-marco-MiniLM-L-6-v2", "cpu")):
        m = f(name, max_length=512, device=device)
        assert isinstance(m, _Original) and m.kwargs == {"max_length": 512, "device": device}
    assert f.original is _Original


def test_served_class_refuses_cpu_and_unknown_activation():
    from marqo_b200.cross_encoder import B200CrossEncoder
    with pytest.raises(ValueError):
        B200CrossEncoder("cross-encoder/ms-marco-TinyBERT-L-2", device="cpu", random_init=1)
    enc = B200CrossEncoder.__new__(B200CrossEncoder)
    enc.num_labels, enc.default_activation_function = 1, torch.nn.Sigmoid()
    assert enc._sigmoid_flag(None) is True and enc._sigmoid_flag(torch.nn.Identity()) is False
    with pytest.raises(ValueError):
        enc._sigmoid_flag(torch.nn.Tanh())
