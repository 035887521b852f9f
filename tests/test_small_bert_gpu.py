"""The 384-wide BERT embedders (MiniLM, e5-small, bge-small: 12 heads of 32) on the GPU: the head_dim-32 instantiations
of both attention kernels vs torch, the encoders vs the CPU fp32 oracle (cosine >= 1 - 1e-3 per vector), and
vectorise() -> GpuTensorIndex at D = 384 vs the oracle and the score oracle."""
import math

import numpy as np
import pytest
import torch

import _checks as K
from oracle import encoders as E

pytestmark = pytest.mark.gpu
MINILM_L6 = E.BertCfg(384, 6, 12, 1536)
E5_SMALL = E.BertCfg(384, 12, 12, 1536)


def _kv_len(g, B, S, mask):
    if mask != 2:
        return None
    kv_len = torch.randint(1, S + 1, (B,), generator=g).to(torch.int32)
    kv_len[0] = S
    return kv_len


def _attention_ref(qkv, B, S, H, mask, kv_len, dtype=torch.float32):
    q, k, v = qkv.to(dtype).view(B, S, 3, H, 32).permute(2, 0, 3, 1, 4)
    att = (q @ k.transpose(-1, -2)) / math.sqrt(32)
    if mask == 1:
        att = att + torch.full((S, S), float("-inf"), dtype=dtype).triu_(1)
    if mask == 2:
        keep = torch.arange(S)[None, :] < kv_len[:, None]
        att = att.masked_fill(~keep[:, None, None, :], float("-inf"))
    return (att.softmax(-1) @ v).permute(0, 2, 1, 3).reshape(B * S, H * 32).float()


# every sequence length around the 64-key (mma.sync) and 128-key (wgmma) block edges, each with all three masks
EDGE_S = [1, 16, 63, 64, 65, 77, 127, 128, 129, 200, 256, 257, 385, 512, 1025]
CASES = [(3, S, 4, mask) for S in EDGE_S for mask in (0, 1, 2)] + [
    # many (batch, head, query block) items, at the 12-head shape of the 384-wide models among them
    (256, 16, 12, 2), (64, 128, 12, 2), (40, 257, 8, 0), (32, 385, 4, 2), (160, 129, 2, 1), (12, 512, 12, 2),
    (100, 65, 6, 0), (90, 77, 12, 1), (8, 1025, 12, 2),
]


@pytest.mark.parametrize("B,S,H,mask", CASES)
def test_attention_hd32_matches_torch(gpu_required, B, S, H, mask):
    from marqo_b200.engine import debug_attention
    g = torch.Generator().manual_seed(B * 1000 + S + 7 * mask)
    W = H * 32
    qkv = K.bf16(torch.randn(B * S, 3 * W, generator=g))
    kv_len = _kv_len(g, B, S, mask)
    ref = _attention_ref(qkv, B, S, H, mask, kv_len)
    got = torch.from_numpy(debug_attention(qkv.numpy(), B, S, W, H, mask, None if kv_len is None else kv_len.numpy()))
    torch.testing.assert_close(got, ref, rtol=2e-2, atol=2e-2)     # P and the output are rounded to bf16
    assert (got - ref).abs().mean() < 3e-3


@pytest.mark.parametrize("B,S,H,mask", [(3, 257, 2, 0), (4, 200, 2, 2), (3, 512, 2, 2), (4, 77, 2, 1), (6, 16, 12, 2),
                                        (3, 129, 12, 1)])
def test_attention_hd32_peaked_scores(gpu_required, B, S, H, mask):
    """Scores with a spread of +-40 (one key dominates most rows): the exponent reference must be the row's true maximum."""
    from marqo_b200.engine import debug_attention
    g = torch.Generator().manual_seed(S + 32)
    W = H * 32
    qkv = torch.randn(B * S, 3 * W, generator=g)
    qkv[:, : 2 * W] *= 3.0                                          # q and k: score std 9, extremes beyond 40
    qkv = K.bf16(qkv)
    kv_len = _kv_len(g, B, S, mask)
    ref = _attention_ref(qkv, B, S, H, mask, kv_len, dtype=torch.float64)
    got = torch.from_numpy(debug_attention(qkv.numpy(), B, S, W, H, mask, None if kv_len is None else kv_len.numpy()))
    assert torch.isfinite(got).all()
    torch.testing.assert_close(got, ref, rtol=3e-2, atol=3e-2)


@pytest.mark.parametrize("hd", [48, 80])
@pytest.mark.parametrize("S", [16, 200])
def test_attention_other_head_dims_are_unsupported(gpu_required, hd, S):
    """W / H outside {32, 64} is refused before any launch, on both the short- and the long-sequence path."""
    from marqo_b200._native import ERR_UNSUPPORTED, NativeError
    from marqo_b200.engine import debug_attention
    H = 4
    qkv = np.zeros((2 * S, 3 * H * hd), np.float32)
    with pytest.raises(NativeError) as ei:
        debug_attention(qkv, 2, S, H * hd, H, 0)
    assert ei.value.code == ERR_UNSUPPORTED


# ------------------------------------------------------------------------------------------------------------------
# Encoders through the C ABI vs the CPU fp32 oracle on the same seeded weights
# ------------------------------------------------------------------------------------------------------------------
def _ids(g, B, S):
    return torch.cat([torch.full((B, 1), 101), torch.randint(1000, 30000, (B, S - 2), generator=g),
                      torch.full((B, 1), 102)], 1)


def test_minilm_l6_batch_256_ragged(gpu_required):
    """all-MiniLM-L6 shape at b256 x 128 tokens (the ingest shape: wgmma attention), ragged key-length masks."""
    from marqo_b200.engine import Encoder
    cfg = MINILM_L6
    sd = E.make_bert_weights(cfg, seed=1234)
    enc = Encoder("bert", E.engine_config(cfg), sd, max_batch=256)
    g = torch.Generator().manual_seed(0)
    ids = _ids(g, 256, 128)
    mask = torch.ones(256, 128, dtype=torch.int64)
    lens = torch.randint(1, 129, (256,), generator=g)
    lens[0], lens[255], lens[100] = 128, 1, 64
    for b in range(256):
        mask[b, int(lens[b]):] = 0
        ids[b, int(lens[b]):] = 0
    got = enc.encode_tokens(ids.numpy(), mask.numpy())
    assert got.shape == (256, 384)
    pos = K.sample_positions(256, 6) + [100]
    K.assert_embeddings_match(got[pos], E.bert_encode(sd, cfg, ids[pos], mask[pos]))
    full = enc.encode_tokens(ids[:4].numpy())                     # no mask: every key counts
    K.assert_embeddings_match(full, E.bert_encode(sd, cfg, ids[:4]))
    enc.close()


def test_e5_small_v2_512_tokens(gpu_required):
    """e5-small-v2 shape at b8 x 512 tokens: full length and ~50 % padded, ragged."""
    from marqo_b200.engine import Encoder
    cfg = E5_SMALL
    sd = E.make_bert_weights(cfg, seed=1234)
    enc = Encoder("bert", E.engine_config(cfg), sd, max_batch=8)
    g = torch.Generator().manual_seed(1)
    ids = _ids(g, 8, 512)
    got = enc.encode_tokens(ids.numpy())
    K.assert_embeddings_match(got[[0, 7]], E.bert_encode(sd, cfg, ids[[0, 7]]))
    mask = torch.ones(8, 512, dtype=torch.int64)
    for b, L in enumerate([256, 200, 312, 256, 1, 511, 256, 300]):
        mask[b, L:] = 0
        ids[b, L:] = 0
    gm = enc.encode_tokens(ids.numpy(), mask.numpy())
    sel = [1, 4, 5]
    K.assert_embeddings_match(gm[sel], E.bert_encode(sd, cfg, ids[sel], mask[sel]))
    enc.close()


@pytest.mark.parametrize("cfg", [MINILM_L6, E5_SMALL], ids=["minilm_l6", "e5_small"])
def test_single_short_query(gpu_required, cfg):
    """b1 x 16 tokens: the search-latency shape (mma.sync attention), eager then replayed from a CUDA graph."""
    from marqo_b200.engine import Encoder
    sd = E.make_bert_weights(cfg, seed=77)
    enc = Encoder("bert", E.engine_config(cfg), sd, max_batch=16)
    g = torch.Generator().manual_seed(2)
    for _ in range(3):
        ids = _ids(g, 1, 16)
        K.assert_embeddings_match(enc.encode_tokens(ids.numpy()), E.bert_encode(sd, cfg, ids))
    ids = _ids(g, 1, 16)
    mask = torch.ones(1, 16, dtype=torch.int64)
    mask[0, 11:] = 0
    ids[0, 11:] = 0
    K.assert_embeddings_match(enc.encode_tokens(ids.numpy(), mask.numpy()), E.bert_encode(sd, cfg, ids, mask))
    enc.close()


# ------------------------------------------------------------------------------------------------------------------
# Through the seams: vectorise("hf/all-MiniLM-L6-v2") -> GpuTensorIndex at D = 384 -> search
# ------------------------------------------------------------------------------------------------------------------
def test_vectorise_minilm_into_index_and_search(gpu_required, score_oracle, monkeypatch):
    from marqo_b200 import model_registry as R, s2_inference as s2, weights as Wt
    s2.clear_loaded_models()
    tok = K.WordTokenizer(101, 102, 1000)
    name = "hf/all-MiniLM-L6-v2"
    props = dict(R.get_model_properties(name), random_init=31, tokenizer=tok)
    rng = np.random.default_rng(3)
    # lengths up to 300 words: sub-batches padded to < 128 (mma.sync) and to >= 128 (wgmma), truncated at 256 tokens
    lengths = np.concatenate([rng.integers(1, 30, size=40), rng.integers(100, 300, size=24)])
    sentences = [" ".join(f"w{int(x)}" for x in rng.integers(0, 28000, size=n)) for n in lengths]
    monkeypatch.setenv("MARQO_MAX_VECTORISE_BATCH_SIZE", "16")          # 4 sub-batches, each padded to its own longest
    out = s2.vectorise(name, sentences, model_properties=props, device="cuda:0", normalize_embeddings=True)
    docs = np.asarray(out, np.float32)
    assert docs.shape == (64, 384)
    sd = {k: torch.from_numpy(v) for k, v in Wt.random_bert_weights(props["arch"], 31).items()}
    ref = []
    for i in range(0, 64, 16):                                           # the reference pads per sub-batch
        t = tok(sentences[i:i + 16], max_length=props["tokens"])
        ref.append(E.bert_encode(sd, MINILM_L6, torch.from_numpy(t["input_ids"]), torch.from_numpy(t["attention_mask"])))
    K.assert_embeddings_match(docs, torch.cat(ref))
    queries = [" ".join(f"w{int(x)}" for x in rng.integers(0, 28000, size=n)) for n in (3, 8, 14)]
    q = np.asarray(s2.vectorise(name, queries, model_properties=props, device="cuda:0", normalize_embeddings=True),
                   np.float32)
    K.assert_embeddings_match(q, E.bert_encode(sd, MINILM_L6, *[torch.from_numpy(v) for v in tok(queries).values()]))
    s2.clear_loaded_models()

    K.assert_index_search_matches(score_oracle, docs, q)
