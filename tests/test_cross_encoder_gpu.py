"""The BERT cross-encoders of Marqo's text reranker on the H100: the BERT embedding with token-type ids and the
sequence-classification head against fp64, the whole forward of TinyBERT-L-2, MiniLM-L-6 and MiniLM-L-12 against the
fp32 oracle (tests/_cross_encoder_oracle.py) on ragged sentence pairs of 16 to 512 tokens, B200CrossEncoder.predict's
contract, the refusals, and the launch count of one classify call."""
import json
import os

import numpy as np
import pytest
import torch

import _cross_encoder_oracle as O
from _checks import COS_TOL, assert_refused, cosine, fp32_oracle  # noqa: F401

pytestmark = pytest.mark.gpu

TINY, L6, L12 = ("cross-encoder/ms-marco-TinyBERT-L-2", "cross-encoder/ms-marco-MiniLM-L-6-v2",
                 "cross-encoder/ms-marco-MiniLM-L-12-v2")
# The bound on |sigmoid score - oracle score| (one label), above the largest differences measured on the H100: 8.7e-3
# in test_model_matches_oracle (MiniLM-L-12, 512 tokens) and 1.8e-2 between predict and transformers in
# tools/rerank_probe.py (MiniLM-L-12, 256 tokens); DESIGN.md §7.5r records both.
SCORE_ATOL = 2e-2
WORDS = ["the", "quick", "brown", "fox", "jump", "over", "lazy", "dog", "hello", "world", "search", "vector", "marqo",
         "is", "a", "re", "rank", "query", "passage", "un", "able", "token", "cafe"]
VOCAB = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + WORDS + ["##s", "##ing", "##ed"] + list("!,.?'-0123456789")


def _pairs(rng, n, S, vocab):
    """n right-padded rows of "[CLS] A [SEP] B [SEP]" with random lengths, the longest S tokens: ids, mask, types."""
    ids = np.zeros((n, S), np.int32)
    mask = np.zeros((n, S), np.int32)
    types = np.zeros((n, S), np.int32)
    for i in range(n):
        L = S if i == 0 else int(rng.integers(3, S + 1))
        la = int(rng.integers(0, L - 2))
        row = [2] + list(rng.integers(5, vocab, la)) + [3] + list(rng.integers(5, vocab, L - 3 - la)) + [3]
        ids[i, :L], mask[i, :L] = row, 1
        types[i, la + 2:L] = 1
    return ids, mask, types


def _model(name, layers=None, labels=None, seed=5, drop=(), max_batch=64):
    """An Encoder of cross-encoder `name` with seeded weights.  labels: the classifier's rows, identity rows first
    when there are more than one (so that the first `width` scores are the pooled rows themselves)."""
    from marqo_b200.engine import Encoder
    a = O.arch(name, **({} if layers is None else {"layers": layers}))
    sd = O.weights(a, seed)
    if labels is not None:
        w = a["width"]
        last = sd["classifier.weight"][:1]
        sd["classifier.weight"] = torch.cat([torch.eye(w), last])[-labels:] if labels > 1 else last
        sd["classifier.bias"] = torch.cat([torch.zeros(w), sd["classifier.bias"][:1]])[-labels:]
        a["num_labels"] = labels
    for k in drop:
        sd.pop(k)
    return a, sd, Encoder("bert", a, sd, max_batch=max_batch)


@pytest.mark.parametrize("w", [128, 384])
def test_embedding_with_type_ids(gpu_required, w):
    from marqo_b200.engine import debug_embed_ln
    rng = np.random.default_rng(w)
    n, S, vocab = 6, 37, 300
    ids, mask, types = _pairs(rng, n, S, vocab)
    word = rng.standard_normal((vocab, w)).astype(np.float32)
    pos = rng.standard_normal((512, w)).astype(np.float32)
    table = rng.standard_normal((2, w)).astype(np.float32)
    g = (1 + 0.1 * rng.standard_normal(w)).astype(np.float32)
    b = (0.1 * rng.standard_normal(w)).astype(np.float32)
    x, h, kv = debug_embed_ln(ids, mask, word, pos, table, g, b, 1e-12, type_ids=types)
    e = word[ids].astype(np.float64) + table[types] + pos[:S]
    mu = e.mean(-1, keepdims=True)
    ref = (e - mu) / np.sqrt(((e - mu) ** 2).mean(-1, keepdims=True) + 1e-12) * g + b
    np.testing.assert_allclose(x, ref.reshape(n * S, w), rtol=0, atol=2e-5)
    np.testing.assert_array_equal(kv, mask.sum(1))
    # all-zero type ids over the table are bit for bit the embedding of today's path (row 0, no type ids)
    x0, h0, _ = debug_embed_ln(ids, mask, word, pos, table[0], g, b, 1e-12)
    xz, hz, _ = debug_embed_ln(ids, mask, word, pos, table, g, b, 1e-12, type_ids=np.zeros_like(types))
    np.testing.assert_array_equal(x0, xz)
    np.testing.assert_array_equal(h0, hz)
    # out-of-range type ids are clamped to the table, as word ids are to the vocabulary
    xc, _, _ = debug_embed_ln(ids, mask, word, pos, table, g, b, 1e-12, type_ids=np.where(types > 0, 7, -3))
    np.testing.assert_array_equal(xc, x)


@pytest.mark.parametrize("w", [128, 384])
@pytest.mark.parametrize("labels", [1, 3])
@pytest.mark.parametrize("sigmoid", [False, True])
def test_head_against_fp64(gpu_required, w, labels, sigmoid):
    from marqo_b200.engine import debug_cls_head
    rng = np.random.default_rng(w + labels)
    n, S = 9, 5   # n not a multiple of the head's 4 sequences per CTA
    x = rng.standard_normal((n * S, w)).astype(np.float32)
    pw = (rng.standard_normal((w, w)) * 1.5 / np.sqrt(w)).astype(np.float32)
    pb = (0.1 * rng.standard_normal(w)).astype(np.float32)
    cw = (rng.standard_normal((labels, w)) * 2 / np.sqrt(w)).astype(np.float32)
    cb = (0.1 * rng.standard_normal(labels)).astype(np.float32)
    got = debug_cls_head(x, S, pw, pb, cw, cb, sigmoid=sigmoid)
    p = np.tanh(x[::S].astype(np.float64) @ pw.T.astype(np.float64) + pb)
    ref = p @ cw.T.astype(np.float64) + cb
    if sigmoid:
        ref = 1 / (1 + np.exp(-ref))
    assert got.shape == (n, labels)
    np.testing.assert_allclose(got, ref, rtol=0, atol=2e-5)


MEASURED = {}


@pytest.mark.parametrize("name,layers", [(TINY, None), (L6, None), (L12, None)], ids=["tinybert-l2", "minilm-l6",
                                                                                       "minilm-l12"])
@pytest.mark.parametrize("S", [16, 128, 512])
def test_model_matches_oracle(gpu_required, name, layers, S):
    a, sd, enc = _model(name, layers, labels=O.arch(name)["width"] + 1)
    try:
        w = a["width"]
        rng = np.random.default_rng(S)
        n = 24 if S < 512 else 8
        ids, mask, types = _pairs(rng, n, S, a["vocab"])
        logits = enc.classify_tokens(ids, mask, types, sigmoid=False)
        scores = enc.classify_tokens(ids, mask, types, sigmoid=True)[:, w]
        dev = torch.device("cuda")
        sdd = {k: v.to(dev) for k, v in sd.items()}
        pooled, ref = (t.cpu() for t in O.forward(sdd, a, *(torch.from_numpy(t.astype(np.int64)).to(dev)
                                                            for t in (ids, mask, types))))
        c = cosine(logits[:, :w], pooled)
        assert float((1 - c).max()) < COS_TOL, f"min cosine {float(c.min())}"
        ref = torch.sigmoid(ref[:, w]).double().numpy()
        err = float(np.abs(scores - ref).max())
        MEASURED[f"{name} S={S}"] = err
        assert err < SCORE_ATOL, f"max |score - oracle| {err}"
        np.testing.assert_allclose(1 / (1 + np.exp(-logits[:, w].astype(np.float64))), scores, rtol=0, atol=1e-6)
        for i in range(n):   # pairs the oracle separates by more than twice the bound keep their order
            far = np.abs(ref - ref[i]) > 2 * SCORE_ATOL
            assert (np.sign(scores[far] - scores[i]) == np.sign(ref[far] - ref[i])).all()
    finally:
        enc.close()
        out = os.environ.get("CROSS_ENCODER_ERR_OUT")   # where to write the differences measured so far
        if out:
            with open(out, "w") as f:
                json.dump(MEASURED, f, indent=1)


@pytest.fixture(scope="module")
def vocab_file(tmp_path_factory):
    p = tmp_path_factory.mktemp("vocab") / "vocab.txt"
    p.write_text("\n".join(VOCAB) + "\n", encoding="utf-8")
    return str(p)


def _texts(rng, n, lo, hi):
    return [" ".join(rng.choice(WORDS, int(rng.integers(lo, hi)))) for _ in range(n)]


def test_predict_contract(gpu_required, vocab_file):
    from marqo_b200.cross_encoder import B200CrossEncoder
    rng = np.random.default_rng(3)
    model = B200CrossEncoder(L6, max_length=512, device="cuda", default_activation_function=torch.nn.Sigmoid(),
                             random_init=9, vocab_file=vocab_file)
    try:
        a = O.arch(L6)
        sd = O.weights(a, 9)
        queries, passages = _texts(rng, 50, 1, 12), _texts(rng, 50, 5, 200)
        pairs = [[" " + q + " ", p + "\n"] for q, p in zip(queries, passages)]
        ref = O.predict(sd, a, model.tokenizer, pairs, 512)
        by_batch = {bs: model.predict(pairs, batch_size=bs) for bs in (1, 32, 1000)}
        for bs, got in by_batch.items():
            assert isinstance(got, np.ndarray) and got.shape == (50,) and got.dtype == np.float32
            np.testing.assert_allclose(got, ref, rtol=0, atol=SCORE_ATOL, err_msg=f"batch_size {bs}")
        one = model.predict(pairs[7])
        assert np.ndim(one) == 0
        np.testing.assert_allclose(one, ref[7], rtol=0, atol=SCORE_ATOL)
        logits = model.predict(pairs[:5], activation_fct=torch.nn.Identity())
        np.testing.assert_allclose(1 / (1 + np.exp(-logits.astype(np.float64))), by_batch[32][:5], rtol=0, atol=1e-6)
        with pytest.raises(ValueError):
            model.predict(pairs[:2], activation_fct=torch.nn.Tanh())
        # Marqo lowers max_length to the tokenizer's (model_utils.py:266-269); predict then truncates there
        model.tokenizer.model_max_length = 64
        if model.max_length > model.tokenizer.model_max_length:
            model.max_length = model.tokenizer.model_max_length
        assert model.max_length == 64
        got = model.predict(pairs)
        np.testing.assert_allclose(got, O.predict(sd, a, model.tokenizer, pairs, 64), rtol=0, atol=SCORE_ATOL)
        assert np.abs(got - ref).max() > SCORE_ATOL   # the truncation changed the long pairs' scores
    finally:
        model.close()


def test_refusals(gpu_required):
    import ctypes as C
    from marqo_b200 import _native as N
    from marqo_b200._native import ERR_INVALID_ARG, ERR_MISSING_WEIGHT, NativeError
    from marqo_b200.engine import Encoder
    from oracle import encoders as E
    a, sd, enc = _model(TINY)
    ids, mask, types = _pairs(np.random.default_rng(0), 2, 16, 1000)
    ids = np.ascontiguousarray(ids)
    try:
        with pytest.raises(NativeError) as e:
            enc.encode_tokens(ids, mask)
        assert e.value.code == ERR_INVALID_ARG
        with pytest.raises(NativeError) as e:   # activation 2 is neither identity nor sigmoid
            N.check(N.load().b200_model_classify_tokens(enc._handle(), ids.ctypes.data, None, None, 2, 16, 2,
                                                        np.empty(2, np.float32).ctypes.data))
        assert e.value.code == ERR_INVALID_ARG
    finally:
        enc.close()
    embedder = Encoder("bert", {k: v for k, v in a.items() if k != "num_labels"},
                       {k[5:]: v for k, v in sd.items() if k.startswith("bert.")}, max_batch=2)
    try:
        with pytest.raises(NativeError) as e:
            embedder.classify_tokens(ids, mask, types)
        assert e.value.code == ERR_INVALID_ARG
    finally:
        embedder.close()
    for missing in (("bert.pooler.dense.weight",), ("classifier.weight", "classifier.bias")):
        s = {k: v for k, v in sd.items() if k not in missing}
        assert_refused("bert", a, s, ERR_MISSING_WEIGHT, missing[0][len("bert."):] if missing[0].startswith("bert.")
                       else missing[0])
    cfg = E.tiny_clip()
    tw = lambda t: dict(width=t.width, layers=t.layers, heads=t.heads, mlp=t.mlp, ctx=t.ctx, vocab=t.vocab,
                        image_size=t.image_size, patch=t.patch)
    d = N.ModelDesc()   # a CLIP model with a classification head
    d.arch, d.embed_dim, d.max_batch, d.cls_labels = N.ARCH_CLIP, cfg.embed_dim, 2, 1
    d.image_std[:] = (1.0, 1.0, 1.0)
    d.vision = N.TowerDesc(*tw(cfg.vision).values())
    d.text = N.TowerDesc(*tw(cfg.text).values())
    h = C.c_void_p()
    assert N.load().b200_model_create(0, C.byref(d), C.byref(h)) == ERR_INVALID_ARG
    assert b"cls_labels" in N.load().b200_last_error()


def test_launch_count_and_graph_replay(gpu_required):
    """The launches one classify call reports (tests/test_model_launches_gpu.py checks the BERT path's count against
    the kernels the device ran): the eager pass, and the CUDA graph its second use captures and later uses replay."""
    a, sd, enc = _model(L6, layers=2)
    ids, mask, types = _pairs(np.random.default_rng(1), 50, 64, a["vocab"])
    try:
        first = enc.classify_tokens(ids, mask, types)   # eager
        # embedding, then per layer QKV, attention, out-projection, LayerNorm, fc1, fc2, LayerNorm, then the head
        assert enc.last_timing()[1] == 1 + 2 * 7 + 1
        for _ in range(2):   # captured, then replayed
            np.testing.assert_array_equal(enc.classify_tokens(ids, mask, types), first)
            assert enc.last_timing()[1] == 1 + 2 * 7 + 1
    finally:
        enc.close()
