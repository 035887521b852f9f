"""multilingual-e5 (XLM-RoBERTa) on the host: the registry entries vs the reference's, the CPU oracle
(tests/_xlmr_oracle.py) vs transformers.XLMRobertaModel, and the C++ SentencePiece Unigram tokenizer vs the
`sentencepiece` library plus fairseq's id offset, on a Unigram model trained by tests/golden/make_unigram_golden.py."""
import json
import unicodedata
from pathlib import Path

import numpy as np
import pytest
import torch

import _xlmr_oracle as X
from marqo_b200 import model_registry as R

GOLDEN_DIR = Path(__file__).resolve().parent / "golden"
MODEL_FILE = GOLDEN_DIR / "unigram_golden.model"
XLMR_NAMES = ("hf/multilingual-e5-small", "hf/multilingual-e5-base", "hf/multilingual-e5-large",
              "hf/multilingual-e5-large-instruct")


# ------------------------------------------------------------------------------------------------------------------
# Registry
# ------------------------------------------------------------------------------------------------------------------
def test_xlmr_entries_are_the_reference_entries():
    ref = json.loads((GOLDEN_DIR / "hf_registry_golden.json").read_text())
    assert sorted(R.XLMR_MODELS) == sorted(XLMR_NAMES)
    for name in XLMR_NAMES:
        entry = R.XLMR_MODELS[name]
        assert {k: v for k, v in entry.items() if k != "arch"} == dict(ref[name], type=R.TYPE_HF), name
        assert R.get_model_properties(name) == entry
        assert R.find_model(name) is entry and R.all_models()[name] is entry
        assert entry["arch"]["width"] == entry["dimensions"]
    assert not set(R.XLMR_MODELS) & set(R.MODELS)


def test_xlmr_arch_blocks():
    for name, (w, layers, heads) in (("hf/multilingual-e5-base", (768, 12, 12)),
                                     ("hf/multilingual-e5-large", (1024, 24, 16)),
                                     ("hf/multilingual-e5-large-instruct", (1024, 24, 16))):
        a = R.XLMR_MODELS[name]["arch"]
        assert a == X.engine_config(X.XlmrCfg(width=w, layers=layers, heads=heads, mlp=4 * w)), name
    small = R.XLMR_MODELS["hf/multilingual-e5-small"]["arch"]
    assert "kind" not in small and small["tokenizer"] == "xlmr"      # a BertModel: the BERT runtime
    assert (small["width"], small["layers"], small["heads"], small["mlp"], small["vocab"], small["max_pos"],
            small["type_vocab"], small["pool"]) == (384, 12, 12, 1536, 250037, 512, 2, "mean")


def test_validate_model_properties_finds_xlmr_by_name():
    from marqo_b200 import s2_inference as s2
    assert s2.validate_model_properties("hf/multilingual-e5-base", None)["arch"]["kind"] == "xlmr"
    custom = s2.validate_model_properties("my-e5", {"name": "intfloat/multilingual-e5-large", "dimensions": 1024,
                                                    "type": "hf"})
    assert custom["arch"] == R.XLMR_MODELS["hf/multilingual-e5-large"]["arch"]


# ------------------------------------------------------------------------------------------------------------------
# The oracle vs transformers.XLMRobertaModel
# ------------------------------------------------------------------------------------------------------------------
def _hf_mean_pool(cfg, sd, ids, mask, normalize=True):
    from transformers import XLMRobertaModel
    m = XLMRobertaModel(X.hf_config(cfg), add_pooling_layer=False).eval()
    res = m.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys and all(k.endswith("_ids") for k in res.missing_keys), res
    with torch.no_grad():
        last = m(input_ids=ids, attention_mask=mask).last_hidden_state
    last = last.masked_fill(~mask[..., None].bool(), 0.0)
    emb = last.sum(dim=1) / mask.sum(dim=1)[..., None]
    return torch.nn.functional.normalize(emb, p=2, dim=1) if normalize else emb


@pytest.mark.parametrize("cfg", [X.tiny_xlmr(), X.XlmrCfg(width=256, layers=2, heads=8, mlp=1024, vocab=3000)],
                         ids=["hd64", "hd32"])
def test_oracle_matches_transformers(cfg):
    """xlmr_encode vs XLMRobertaModel (eager, fp32, dropout 0): rows of 1, 40 and 512 tokens, right padding, and a
    pad id inside the text (its position is the pad's and later tokens shift down)."""
    sd = X.make_xlmr_weights(cfg, seed=21)
    g = torch.Generator().manual_seed(5)
    ids, mask = X.ragged_ids(g, 5, 512, [1, 40, 512, 300, 7], cfg.vocab)
    ids[3, 100] = cfg.pad_id
    for normalize in (True, False):
        got = X.xlmr_encode(sd, cfg, ids, mask, normalize=normalize)
        want = _hf_mean_pool(cfg, sd, ids, mask, normalize=normalize)
        torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-5)


def test_oracle_position_ids_follow_the_ids():
    ids = torch.tensor([[0, 7, 1, 9, 2, 1, 1]])
    assert X.position_ids(ids, 1).tolist() == [[2, 3, 1, 4, 5, 1, 1]]
    from transformers.models.xlm_roberta.modeling_xlm_roberta import XLMRobertaEmbeddings
    assert XLMRobertaEmbeddings.create_position_ids_from_input_ids(ids, 1).tolist() == X.position_ids(ids, 1).tolist()


# ------------------------------------------------------------------------------------------------------------------
# The Unigram tokenizer vs sentencepiece
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sp():
    spm = pytest.importorskip("sentencepiece")
    return spm.SentencePieceProcessor(model_file=str(MODEL_FILE))


@pytest.fixture(scope="module")
def tok(native_lib):
    from marqo_b200.tokenizers import XLMRTokenizer
    return XLMRTokenizer(str(MODEL_FILE))


def _ours(tok, texts, max_length=100000):
    out = tok(texts, padding=True, truncation=True, max_length=max_length)
    return [row[m == 1].tolist() for row, m in zip(out["input_ids"], out["attention_mask"])]


def _assert_same(tok, sp, texts, max_length=100000):
    got = _ours(tok, texts, max_length)
    bad = [(t, g, X.fairseq_ids(sp, t)) for t, g in zip(texts, got) if g != X.fairseq_ids(sp, t)]
    assert not bad, f"{len(bad)} of {len(texts)} differ, first: {bad[:3]}"


def _assigned(lo, hi):
    return [chr(c) for c in range(lo, hi) if not 0xD800 <= c <= 0xDFFF and unicodedata.category(chr(c)) != "Cn"]


def test_every_assigned_code_point(tok, sp):
    """One string per assigned code point of the BMP and the supplementary planes 1-3 (every assigned block but the
    two supplementary private-use planes), plus each 64-code-point run of them as one string."""
    cps = _assigned(0, 0x40000) + _assigned(0xE0000, 0xE0200)
    assert len(cps) > 150000
    _assert_same(tok, sp, cps)
    _assert_same(tok, sp, ["".join(cps[i:i + 64]) for i in range(0, len(cps), 64)])


def test_nfkc_accents_scripts(tok, sp):
    texts = ["ﬁne ﬂow", "ＡＢＣ ａｂｃ １２３", "①②③ ⑳", "ｶﾀｶﾅ ﾊﾟ", "㎞ ㍿ Ⅻ ½", "café naïve Ångström ñandú",
             "é ä ñ", "東京大学で日本語を学ぶ", "中文字 学生先生", "Привет мир, как дела?",
             "αβγ Ωμέγα", "mixed 東京 мир ﬁ Ａ①", "ß ẞ İ ı", "x​zero­width﻿", "emoji 😀👍🏽 and ☃☃☃"]
    _assert_same(tok, sp, texts)


def test_whitespace(tok, sp):
    texts = ["", " ", "   ", "\t", "\n\n", " \t\n ", "a  b", "a\tb\nc\r\nd", "  leading", "trailing   ",
             "  both  ends  ", "many     inner      spaces", "　ideographic　space", "nbsp here",
             "▁already escaped▁", "tab\t\t\tthen"]
    _assert_same(tok, sp, texts)


def test_truncation_keeps_the_end_token(tok, sp):
    text = "東京大学 " * 200 + "абв"
    full = X.fairseq_ids(sp, text)
    assert len(full) > 128
    for L in (2, 3, 128, 512):
        got = _ours(tok, [text], max_length=L)[0]
        assert got == full[:L - 1] + [2], L


def test_batch_padding(tok, sp):
    texts = ["short", "a much longer sentence with 東京 and мир in it", "", "mid length text"]
    out = tok(texts, padding=True, truncation=True, max_length=512, return_tensors="np")
    assert set(out) == {"input_ids", "attention_mask"}
    ids, mask = out["input_ids"], out["attention_mask"]
    assert ids.dtype == np.int64 and mask.dtype == np.int64
    want = [X.fairseq_ids(sp, t) for t in texts]
    assert ids.shape == (4, max(len(w) for w in want))
    for row, m, w in zip(ids, mask, want):
        n = len(w)
        assert row[:n].tolist() == w and (row[n:] == 1).all()
        assert m[:n].tolist() == [1] * n and (m[n:] == 0).all()
    single = tok("short", return_tensors="pt")
    assert single["input_ids"].tolist() == [want[0]]


def test_vocab_size_and_threads(tok, sp):
    assert tok.vocab_size == sp.get_piece_size() + 2          # + <pad> and <mask>
    texts = [f"line {i} 東京 мир " * (i % 7 + 1) for i in range(257)]   # enough rows for the thread pool
    _assert_same(tok, sp, texts)


def test_refuses_non_unigram_models(native_lib):
    pb = pytest.importorskip("sentencepiece.sentencepiece_model_pb2")
    from marqo_b200._native import ERR_INVALID_ARG, ERR_UNSUPPORTED, NativeError
    from marqo_b200.tokenizers import XLMRTokenizer
    m = pb.ModelProto()
    m.ParseFromString(MODEL_FILE.read_bytes())
    m.trainer_spec.model_type = pb.TrainerSpec.BPE
    with pytest.raises(NativeError) as ei:
        XLMRTokenizer(m.SerializeToString())
    assert ei.value.code == ERR_UNSUPPORTED
    with pytest.raises(NativeError) as ei:
        XLMRTokenizer(MODEL_FILE.read_bytes()[:1000])
    assert ei.value.code == ERR_INVALID_ARG


def test_hf_loader_picks_the_unigram_tokenizer(native_lib, tmp_path):
    from marqo_b200.loaders import B200HuggingFace
    from marqo_b200.tokenizers import XLMRTokenizer, is_sentencepiece_model
    assert is_sentencepiece_model(str(MODEL_FILE)) and is_sentencepiece_model(MODEL_FILE.read_bytes())
    vocab = tmp_path / "vocab.txt"
    vocab.write_text("[PAD]\n[UNK]\n[CLS]\n[SEP]\n")
    assert not is_sentencepiece_model(str(vocab)) and not is_sentencepiece_model(vocab.read_bytes())
    for name in ("hf/multilingual-e5-small", "hf/multilingual-e5-base"):
        m = B200HuggingFace(device="cpu", model_properties=dict(R.get_model_properties(name), vocab_file=str(MODEL_FILE)))
        m.arch = m.model_properties["arch"]
        assert isinstance(m._default_tokenizer(), XLMRTokenizer), name
