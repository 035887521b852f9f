"""MPNet on the GPU: both attention kernels with the relative-position bias vs torch, the MPNet-base encoder vs the CPU
fp32 oracle (cosine >= 1 - 1e-3, unit norm), the reference's golden vectors through the C ABI, and
vectorise("hf/all-mpnet-base-v2") with the C++ tokenizer -> GpuTensorIndex vs the oracle and the score oracle."""
import math

import numpy as np
import pytest
import torch

import _checks as K
import _mpnet_oracle as M

pytestmark = pytest.mark.gpu
BASE = M.MPNET_BASE


def _attention_ref(qkv, B, S, H, kv_len, bias):
    q, k, v = qkv.double().view(B, S, 3, H, 64).permute(2, 0, 3, 1, 4)
    smax = (bias.shape[1] + 1) // 2
    rel = torch.arange(S)[None, :] - torch.arange(S)[:, None] + smax - 1
    att = (q @ k.transpose(-1, -2)) / 8.0 + bias.double()[:, rel][None]
    keep = torch.arange(S)[None, :] < kv_len[:, None]
    att = att.masked_fill(~keep[:, None, None, :], float("-inf"))
    return (att.softmax(-1) @ v).permute(0, 2, 1, 3).reshape(B * S, H * 64).float()


@pytest.mark.parametrize("S", [1, 16, 63, 64, 65, 127, 128, 129, 257, 512])
@pytest.mark.parametrize("peaked", [False, True], ids=["plain", "peaked"])
def test_attention_rel_bias_matches_torch(gpu_required, S, peaked):
    """S < 128 runs the mma.sync kernel, S >= 128 the wgmma one; key lengths ragged; bias values up to +-20."""
    from marqo_b200.engine import debug_attention
    g = torch.Generator().manual_seed(S + 1000 * peaked)
    B, H, smax = 3, 4, 512
    qkv = torch.randn(B * S, 3 * H * 64, generator=g)
    if peaked:
        qkv[:, : 2 * H * 64] *= 3.0                                  # score std 9: one key dominates most rows
    qkv = K.bf16(qkv)
    bias = (torch.rand(H, 2 * smax - 1, generator=g) * 40 - 20) if peaked else torch.randn(H, 2 * smax - 1, generator=g)
    kv_len = torch.randint(1, S + 1, (B,), generator=g).to(torch.int32)
    kv_len[0] = S
    got = torch.from_numpy(debug_attention(qkv.numpy(), B, S, H * 64, H, 2, kv_len.numpy(), rel_bias=bias.numpy()))
    ref = _attention_ref(qkv, B, S, H, kv_len, bias)
    assert torch.isfinite(got).all()
    torch.testing.assert_close(got, ref, rtol=3e-2, atol=3e-2)     # P and the output are rounded to bf16
    assert (got - ref).abs().mean() < 4e-3


def test_attention_rel_bias_refuses_longer_sequences_than_the_table(gpu_required):
    from marqo_b200._native import ERR_INVALID_ARG, NativeError
    from marqo_b200.engine import debug_attention
    qkv = np.zeros((2 * 200, 3 * 128), np.float32)
    with pytest.raises(NativeError) as ei:
        debug_attention(qkv, 2, 200, 128, 2, 2, np.full(2, 200, np.int32), rel_bias=np.zeros((2, 2 * 100 - 1), np.float32))
    assert ei.value.code == ERR_INVALID_ARG


# ------------------------------------------------------------------------------------------------------------------
# The encoder through the C ABI vs the CPU fp32 oracle on the same seeded weights
# ------------------------------------------------------------------------------------------------------------------
def _ids(g, B, S, lens=None):
    ids = torch.randint(5, 30000, (B, S), generator=g)
    ids[:, 0] = 0
    mask = torch.ones(B, S, dtype=torch.int64)
    for b in range(B):
        L = S if lens is None else int(lens[b])
        ids[b, L - 1] = 2
        ids[b, L:] = BASE.pad_id
        mask[b, L:] = 0
    return ids, mask


@pytest.fixture(scope="module")
def base_weights():
    return M.make_mpnet_weights(BASE, seed=1234)


def test_mpnet_base_batch_256_ragged(gpu_required, base_weights):
    """b256 x 128 tokens (wgmma attention), ragged masks, one row with the pad id inside the text."""
    from marqo_b200.engine import Encoder
    enc = Encoder("mpnet", M.engine_config(BASE), base_weights, max_batch=256)
    g = torch.Generator().manual_seed(0)
    lens = torch.randint(1, 129, (256,), generator=g)
    lens[0], lens[255], lens[100] = 128, 1, 64
    ids, mask = _ids(g, 256, 128, lens)
    ids[100, 20] = BASE.pad_id
    got = enc.encode_tokens(ids.numpy(), mask.numpy())
    assert got.shape == (256, 768)
    pos = [0, 1, 37, 100, 200, 254, 255]
    K.assert_embeddings_match(got[pos], M.mpnet_encode(base_weights, BASE, ids[pos], mask[pos]))
    enc.close()


def test_mpnet_base_512_tokens_and_513_refused(gpu_required, base_weights):
    """b8 x 512 tokens, the longest sequence MPNet-base takes; 513 is refused."""
    from marqo_b200._native import ERR_INVALID_ARG, NativeError
    from marqo_b200.engine import Encoder
    enc = Encoder("mpnet", M.engine_config(BASE), base_weights, max_batch=8)
    g = torch.Generator().manual_seed(1)
    ids, mask = _ids(g, 8, 512, [512, 200, 312, 256, 1, 511, 256, 300])
    got = enc.encode_tokens(ids.numpy(), mask.numpy())
    sel = [0, 1, 4, 5]
    K.assert_embeddings_match(got[sel], M.mpnet_encode(base_weights, BASE, ids[sel], mask[sel]))
    with pytest.raises(NativeError) as ei:
        enc.encode_tokens(np.zeros((1, 513), np.int32))
    assert ei.value.code == ERR_INVALID_ARG
    enc.close()


def test_mpnet_base_single_query_graph_replay(gpu_required, base_weights):
    """b1 x 16 (mma.sync attention) three times: eager, captured, replayed from the CUDA graph."""
    from marqo_b200.engine import Encoder
    enc = Encoder("mpnet", M.engine_config(BASE), base_weights, max_batch=16)
    g = torch.Generator().manual_seed(2)
    for i in range(3):
        ids, mask = _ids(g, 1, 16, [16 - 3 * i])
        K.assert_embeddings_match(enc.encode_tokens(ids.numpy(), mask.numpy()),
                                  M.mpnet_encode(base_weights, BASE, ids, mask))
    enc.close()


def test_missing_relative_attention_bias(gpu_required):
    from marqo_b200._native import ERR_MISSING_WEIGHT
    cfg = M.tiny_mpnet()
    sd = M.make_mpnet_weights(cfg, seed=3)
    del sd["encoder.relative_attention_bias.weight"]
    K.assert_refused("mpnet", M.engine_config(cfg), sd, ERR_MISSING_WEIGHT)


def test_golden_vectors_through_the_c_abi(gpu_required):
    """The reference's HuggingFaceModel.encode on MPNetModel (tests/golden/make_mpnet_golden.py) vs the engine."""
    from pathlib import Path
    from marqo_b200.engine import Encoder
    z = np.load(Path(__file__).resolve().parent / "golden" / "mpnet_golden.npz")
    cfg = M.tiny_mpnet()
    enc = Encoder("mpnet", M.engine_config(cfg), M.make_mpnet_weights(cfg, seed=int(z["seed"])), max_batch=8)
    K.assert_embeddings_match(enc.encode_tokens(z["ids"], z["mask"]), z["vec"])
    un = enc.encode_tokens(z["ids"], z["mask"], normalize=False)
    K.assert_embeddings_match(un, z["vec_unnormalized"], unit_norm=False)
    np.testing.assert_allclose(np.linalg.norm(un, axis=1), np.linalg.norm(z["vec_unnormalized"], axis=1), rtol=1e-2)
    enc.close()


# ------------------------------------------------------------------------------------------------------------------
# Through the seams: vectorise("hf/all-mpnet-base-v2") with the C++ tokenizer -> GpuTensorIndex -> search
# ------------------------------------------------------------------------------------------------------------------
def test_vectorise_mpnet_into_index_and_search(gpu_required, score_oracle, monkeypatch, tmp_path):
    from transformers import MPNetTokenizer as HF
    from marqo_b200 import model_registry as R, s2_inference as s2, weights as Wt
    s2.clear_loaded_models()
    vf = tmp_path / "vocab.txt"
    vocab = M.synthetic_vocab(30527)
    vf.write_text("\n".join(vocab) + "\n")
    name = "hf/all-mpnet-base-v2"
    props = dict(R.get_model_properties(name), random_init=31, vocab_file=str(vf))
    rng = np.random.default_rng(3)
    words = vocab[9:-1]
    lengths = np.concatenate([rng.integers(1, 30, size=40), rng.integers(100, 200, size=24)])
    sentences = [" ".join(words[int(x)] for x in rng.integers(0, len(words), size=n)) for n in lengths]
    sentences[5] += " <pad> <mask> [CLS]"
    monkeypatch.setenv("MARQO_MAX_VECTORISE_BATCH_SIZE", "16")
    out = s2.vectorise(name, sentences, model_properties=props, device="cuda:0", normalize_embeddings=True)
    docs = np.asarray(out, np.float32)
    assert docs.shape == (64, 768)
    sd = {k: torch.from_numpy(v) for k, v in Wt.random_mpnet_weights(props["arch"], 31).items()}
    hf = HF(str(vf))
    ref = []
    for i in range(0, 64, 16):                                           # the reference pads per sub-batch
        t = hf(sentences[i:i + 16], padding=True, truncation=True, max_length=props["tokens"], return_tensors="pt")
        ref.append(M.mpnet_encode(sd, BASE, t["input_ids"], t["attention_mask"]))
    K.assert_embeddings_match(docs, torch.cat(ref))
    queries = [" ".join(words[int(x)] for x in rng.integers(0, len(words), size=n)) for n in (3, 8, 14)]
    q = np.asarray(s2.vectorise(name, queries, model_properties=props, device="cuda:0", normalize_embeddings=True),
                   np.float32)
    t = hf(queries, padding=True, truncation=True, max_length=props["tokens"], return_tensors="pt")
    K.assert_embeddings_match(q, M.mpnet_encode(sd, BASE, t["input_ids"], t["attention_mask"]))
    s2.clear_loaded_models()

    K.assert_index_search_matches(score_oracle, docs, q)
