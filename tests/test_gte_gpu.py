"""The Stella embedder (GTE encoder) on the GPU: the full 24 layers at b16 x 512 with ragged lengths against the fp32
oracle (cosine >= 1 - 1e-3, unit norm), a single 16-token query through the eager, captured and replayed graph paths,
the refusals, and vectorise(stella) with the C++ WordPiece tokenizer ->
GpuTensorIndex against the score oracle.  The oracle runs on the GPU in fp32 with TF32 off.  The launch count at
2 layers is in tests/test_model_launches_gpu.py and device memory after close in tests/test_device_memory_gpu.py."""
import numpy as np
import pytest
import torch

import _gte_oracle as G
from _checks import (assert_embeddings_match, assert_index_search_matches, assert_refused, cosine,
                     fp32_oracle)  # noqa: F401 (fp32_oracle: autouse)
from marqo_b200._native import ERR_INVALID_ARG, ERR_MISSING_WEIGHT, NativeError

pytestmark = pytest.mark.gpu


def _encoder(cfg, sd, max_batch):
    from marqo_b200.engine import Encoder
    return Encoder("gte", G.engine_config(cfg), sd, max_batch=max_batch)


def _ref(sd, cfg, ids, mask, normalize=True):
    return G.gte_encode({k: v.cuda() for k, v in sd.items()}, cfg, ids, mask, normalize=normalize).cpu()


def test_full_depth_ragged_b16x512(gpu_required):
    """24 layers at the real shape: lengths 1 .. 512, one row full and one a lone [CLS]."""
    cfg = G.STELLA
    sd = G.make_gte_weights(cfg, seed=11)
    enc = _encoder(cfg, sd, 16)
    try:
        g = torch.Generator().manual_seed(0)
        lens = torch.randint(2, 512, (16,), generator=g)
        lens[0], lens[1], lens[2] = 512, 1, 129
        ids, mask = G.ragged_ids(g, lens.tolist(), 512, cfg.vocab)
        ids[3, 7] = cfg.vocab - 1
        got = enc.encode_tokens(ids.numpy(), mask.numpy())
        assert got.shape == (16, 1024)
        raw = enc.encode_tokens(ids[:2].numpy(), mask[:2].numpy(), normalize=False)
    finally:
        enc.close()   # the device memory goes to the fp32 oracle
    ref = _ref(sd, cfg, ids, mask)
    print(f"\n[gte full depth] b16 x 512: worst cosine {float(cosine(got, ref).min()):.6f}")
    assert_embeddings_match(got, ref)
    assert_embeddings_match(raw, _ref(sd, cfg, ids[:2], mask[:2], normalize=False), unit_norm=False)


def test_new_prefix_is_dropped(gpu_required):
    cfg = G.tiny_gte()
    sd = G.make_gte_weights(cfg, seed=3)
    enc = _encoder(cfg, {"new." + k: v for k, v in sd.items()}, 4)
    try:
        ids, mask = G.ragged_ids(torch.Generator().manual_seed(1), [64, 1, 33, 10], 64, cfg.vocab)
        assert_embeddings_match(enc.encode_tokens(ids.numpy(), mask.numpy()), _ref(sd, cfg, ids, mask))
    finally:
        enc.close()


def test_single_query_graph_path(gpu_required):
    """A single 16-token query runs eagerly once, is captured into a CUDA graph on the second call and replayed after:
    every call gives the bits of the first, which match the oracle."""
    cfg = G.GteCfg(layers=2)
    sd = G.make_gte_weights(cfg, seed=5)
    enc = _encoder(cfg, sd, 4)
    try:
        ids, mask = G.ragged_ids(torch.Generator().manual_seed(2), [16], 16, cfg.vocab)
        runs = [enc.encode_tokens(ids.numpy(), mask.numpy()) for _ in range(4)]
        for r in runs[1:]:
            np.testing.assert_array_equal(r, runs[0])
        # embed, 2 layers x (QKV, rope, attention, o_proj, attn_ln, up_gate, geglu, down, mlp_ln), the head
        assert enc.last_timing()[1] == 1 + 2 * 9 + 1
        assert_embeddings_match(runs[0], _ref(sd, cfg, ids, mask))
    finally:
        enc.close()


# ------------------------------------------------------------------------------------------------------------------
# Refusals
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["head_dim_32", "width_1280", "ctx_1024", "no_eps", "no_theta", "ntk_below_1"])
def test_bad_shapes_are_refused_at_create(gpu_required, case):
    a = G.engine_config(G.GteCfg(layers=1))
    a.update({"head_dim_32": dict(heads=32), "width_1280": dict(width=1280, heads=20), "ctx_1024": dict(ctx=1024),
              "no_eps": dict(ln_eps=0.0), "no_theta": dict(rope_theta=0.0), "ntk_below_1": dict(rope_ntk_factor=0.5)
              }[case])
    assert_refused("gte", a, {}, ERR_INVALID_ARG)


def test_missing_weight_wrong_up_gate_and_long_sequence(gpu_required):
    cfg = G.tiny_gte()
    a, sd = G.engine_config(cfg), G.make_gte_weights(cfg, seed=6)
    missing = {k: v for k, v in sd.items() if k != "encoder.layer.1.mlp_ln.bias"}
    assert_refused("gte", a, missing, ERR_MISSING_WEIGHT, "mlp_ln.bias")
    # an up_gate_proj of mlp rows (no gate half)
    wrong = dict(sd)
    wrong["encoder.layer.0.mlp.up_gate_proj.weight"] = sd["encoder.layer.0.mlp.up_gate_proj.weight"][:cfg.mlp]
    assert_refused("gte", a, wrong, ERR_INVALID_ARG)
    enc = _encoder(cfg, sd, 2)
    try:
        with pytest.raises(NativeError) as e:
            enc.encode_tokens(np.zeros((1, cfg.ctx + 1), np.int32))
        assert e.value.code == ERR_INVALID_ARG
    finally:
        enc.close()


# ------------------------------------------------------------------------------------------------------------------
# Through the seams: vectorise -> GpuTensorIndex -> search
# ------------------------------------------------------------------------------------------------------------------
def test_vectorise_stella_into_index_and_search(gpu_required, score_oracle, tmp_path, monkeypatch):
    from marqo_b200 import model_registry as R, s2_inference as s2
    from oracle import tokenizers as OT
    words = ["alpha", "beta", "gamma", "delta", "search", "vector", "index", "query", "stella", "model", "##s", "##ing"]
    vocab = (["[PAD]"] + [f"[unused{i}]" for i in range(99)] + ["[UNK]", "[CLS]", "[SEP]", "[MASK]"] + words
             + [f"w{i}" for i in range(400)])
    path = tmp_path / "vocab.txt"
    path.write_text("\n".join(vocab) + "\n")
    s2.clear_loaded_models()
    props = dict(R.get_model_properties(G.NAME), random_init=23, vocab_file=str(path), max_batch=16)
    props["arch"]["layers"] = 2
    rng = np.random.default_rng(5)
    pool = words[:10] + [f"w{i}" for i in range(400)] + ["unknownword", "searching", "models"]
    texts = [" ".join(pool[int(i)] for i in rng.integers(0, len(pool), int(n)))
             for n in rng.integers(1, 700, 40)]
    monkeypatch.setenv("MARQO_MAX_VECTORISE_BATCH_SIZE", "16")
    docs = np.asarray(s2.vectorise(G.NAME, texts, model_properties=props, device="cuda:0", normalize_embeddings=True),
                      np.float32)
    assert docs.shape == (40, 1024)
    queries = np.asarray(s2.vectorise(G.NAME, ["alpha search", "vector index", "stella models"],
                                      model_properties=props, device="cuda:0", normalize_embeddings=True), np.float32)
    s2.clear_loaded_models()
    cfg = G.GteCfg(layers=2)
    sd = G.make_gte_weights(cfg, seed=23)
    sel = [0, 7, 39]
    ids, mask = OT.bert_encode_batch(OT.bert_wordpiece(vocab), [texts[i] for i in sel], 512)
    assert (ids[:, 0] == 101).all() and ids.shape[1] <= 512
    assert_embeddings_match(docs[sel], _ref(sd, cfg, torch.from_numpy(ids), torch.from_numpy(mask)))
    assert_index_search_matches(score_oracle, docs, queries)
