"""multilingual-e5 on the GPU: the XLM-R encoder through the C ABI vs the CPU fp32 oracle on the same seeded weights
(cosine >= 1 - 1e-3 per vector, unit norm) at the base and large shapes, multilingual-e5-small's BertModel on the BERT
runtime, the refusals, and vectorise("hf/multilingual-e5-base") with the C++ Unigram tokenizer -> GpuTensorIndex vs the
score oracle."""
from pathlib import Path

import numpy as np
import pytest
import torch

import _checks as K
import _xlmr_oracle as X

pytestmark = pytest.mark.gpu
MODEL_FILE = Path(__file__).resolve().parent / "golden" / "unigram_golden.model"


def _encoder(cfg, sd, max_batch):
    from marqo_b200.engine import Encoder
    return Encoder("xlmr", X.engine_config(cfg), sd, max_batch=max_batch)


def test_xlmr_base_full_depth_ragged(gpu_required):
    """XLM-R base, 12 layers, b16 x 512: lengths 1 .. 512, right padding, one pad id inside the text; the ids span the
    whole 250002-row word table."""
    cfg = X.XLMR_BASE
    sd = X.make_xlmr_weights(cfg, seed=11)
    enc = _encoder(cfg, sd, 16)
    g = torch.Generator().manual_seed(0)
    lens = torch.randint(2, 512, (16,), generator=g)
    lens[0], lens[1], lens[2], lens[3] = 512, 1, 40, 511
    ids, mask = X.ragged_ids(g, 16, 512, lens, cfg.vocab)
    ids[1, 0] = 2                                           # a one-token row
    ids[4, 10] = cfg.pad_id
    ids[5, 3] = cfg.vocab - 1
    got = enc.encode_tokens(ids.numpy(), mask.numpy())
    assert got.shape == (16, 768)
    sel = [0, 1, 2, 3, 4, 5, 15]
    K.assert_embeddings_match(got[sel], X.xlmr_encode(sd, cfg, ids[sel], mask[sel]))
    enc.close()


def test_xlmr_large_two_layers_b64(gpu_required):
    """The large shape (width 1024, 16 heads) at 2 layers, b64 x 512."""
    cfg = X.XlmrCfg(width=1024, layers=2, heads=16, mlp=4096)
    sd = X.make_xlmr_weights(cfg, seed=12)
    enc = _encoder(cfg, sd, 64)
    g = torch.Generator().manual_seed(1)
    lens = torch.randint(1, 513, (64,), generator=g)
    lens[0], lens[63] = 512, 1
    ids, mask = X.ragged_ids(g, 64, 512, lens, cfg.vocab)
    ids[63, 0] = 2
    got = enc.encode_tokens(ids.numpy(), mask.numpy())
    assert got.shape == (64, 1024)
    sel = [0, 17, 40, 63]
    K.assert_embeddings_match(got[sel], X.xlmr_encode(sd, cfg, ids[sel], mask[sel]))
    enc.close()


def test_xlmr_large_full_depth_and_513_refused(gpu_required):
    """multilingual-e5-large's full 24 layers at b8 x 512; 513 tokens are refused."""
    from marqo_b200._native import ERR_INVALID_ARG, NativeError
    cfg = X.XLMR_LARGE
    sd = X.make_xlmr_weights(cfg, seed=13)
    enc = _encoder(cfg, sd, 8)
    g = torch.Generator().manual_seed(2)
    ids, mask = X.ragged_ids(g, 8, 512, [512, 100, 512, 37, 256, 511, 3, 400], cfg.vocab)
    got = enc.encode_tokens(ids.numpy(), mask.numpy())
    sel = [0, 3]
    K.assert_embeddings_match(got[sel], X.xlmr_encode(sd, cfg, ids[sel], mask[sel]))
    with pytest.raises(NativeError) as ei:
        enc.encode_tokens(np.zeros((1, 513), np.int32))
    assert ei.value.code == ERR_INVALID_ARG
    enc.close()


def test_xlmr_small_runs_the_bert_runtime(gpu_required):
    """multilingual-e5-small is a BertModel over the 250037-piece XLM-R vocabulary (absolute positions, eps 1e-12)."""
    from oracle.encoders import BertCfg, bert_encode
    from marqo_b200 import model_registry as R, weights as Wt
    from marqo_b200.engine import Encoder
    arch = R.XLMR_MODELS["hf/multilingual-e5-small"]["arch"]
    sd = {k: torch.from_numpy(v) for k, v in Wt.random_bert_weights(arch, 14).items()}
    enc = Encoder("bert", arch, sd, max_batch=16)
    g = torch.Generator().manual_seed(3)
    ids, mask = X.ragged_ids(g, 16, 512, [512, 1, 40, 300] + [200] * 12, arch["vocab"])
    ids[1, 0] = 2
    ids[2, 5] = arch["vocab"] - 1
    got = enc.encode_tokens(ids.numpy(), mask.numpy())
    cfg = BertCfg(384, 12, 12, 1536, vocab=250037, max_pos=512, type_vocab=2)
    sel = [0, 1, 2, 3]
    K.assert_embeddings_match(got[sel], bert_encode(sd, cfg, ids[sel], mask[sel]))
    enc.close()


def test_roberta_prefix_and_missing_type_row(gpu_required):
    from marqo_b200._native import ERR_MISSING_WEIGHT
    cfg = X.tiny_xlmr()
    sd = X.make_xlmr_weights(cfg, seed=15)
    enc = _encoder(cfg, {"roberta." + k: v for k, v in sd.items()}, 4)
    g = torch.Generator().manual_seed(4)
    ids, mask = X.ragged_ids(g, 4, 64, [64, 1, 33, 10], cfg.vocab)
    ids[1, 0] = 2
    K.assert_embeddings_match(enc.encode_tokens(ids.numpy(), mask.numpy()), X.xlmr_encode(sd, cfg, ids, mask))
    enc.close()
    del sd["embeddings.token_type_embeddings.weight"]
    K.assert_refused("xlmr", X.engine_config(cfg), sd, ERR_MISSING_WEIGHT)


# ------------------------------------------------------------------------------------------------------------------
# Through the seams: vectorise("hf/multilingual-e5-base") with the Unigram tokenizer -> GpuTensorIndex -> search
# ------------------------------------------------------------------------------------------------------------------
def test_vectorise_multilingual_e5_into_index_and_search(gpu_required, score_oracle, monkeypatch):
    import sentencepiece as spm
    from marqo_b200 import model_registry as R, s2_inference as s2
    s2.clear_loaded_models()
    name = "hf/multilingual-e5-base"
    props = dict(R.get_model_properties(name), random_init=41, vocab_file=str(MODEL_FILE))
    sp = spm.SentencePieceProcessor(model_file=str(MODEL_FILE))
    rng = np.random.default_rng(4)
    alphabet = "abcdefghijklmnopqrstuvwxyzéñü東京大学日本語абвгдежзαβγ ①Ａﬁ"
    lengths = np.concatenate([rng.integers(1, 60, size=40), rng.integers(300, 900, size=24)])
    sentences = ["".join(alphabet[int(x)] for x in rng.integers(0, len(alphabet), size=n)) for n in lengths]
    sentences[3] = "   "
    monkeypatch.setenv("MARQO_MAX_VECTORISE_BATCH_SIZE", "16")
    out = s2.vectorise(name, sentences, model_properties=props, device="cuda:0", normalize_embeddings=True)
    docs = np.asarray(out, np.float32)
    assert docs.shape == (64, 768)
    cfg = X.XLMR_BASE
    sd = X.make_xlmr_weights(cfg, seed=41)

    def oracle(texts):
        rows = [X.fairseq_ids(sp, t) for t in texts]
        rows = [r if len(r) <= 512 else r[:511] + [2] for r in rows]
        L = max(len(r) for r in rows)
        ids = torch.tensor([r + [1] * (L - len(r)) for r in rows])
        mask = torch.tensor([[1] * len(r) + [0] * (L - len(r)) for r in rows])
        return X.xlmr_encode(sd, cfg, ids, mask)

    sel = [0, 3, 17, 39, 40, 63]
    K.assert_embeddings_match(docs[sel], oracle([sentences[i] for i in sel]))
    queries = ["東京 大学", "привет мир", "ﬁne café", "αβγ"]
    q = np.asarray(s2.vectorise(name, queries, model_properties=props, device="cuda:0", normalize_embeddings=True),
                   np.float32)
    K.assert_embeddings_match(q, oracle(queries))
    s2.clear_loaded_models()

    K.assert_index_search_matches(score_oracle, docs, q)
