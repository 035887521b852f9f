"""The M-CLIP models on the GPU: the projected text head against fp64 at every served width -> dimensions, with key
lengths 1, 129 and 512 and normalize on and off; both text towers through the C ABI against the fp32 oracle (cosine
>= 1 - 1e-3), LaBSE at full depth over its whole 501153-row vocabulary; the image vectors bit for bit against
B200Clip's on the same weights; launch counts against the plain XLM-R tower; device memory after close; 513 tokens
refused with nothing written; and vectorise("multilingual-clip/XLM-Roberta-Large-Vit-B-32") on text and images ->
GpuTensorIndex -> search against the score oracle."""
import ctypes
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import _mclip_oracle as M
import _xlmr_oracle as X
from _checks import assert_embeddings_match, assert_index_search_matches, fp32_oracle  # noqa: F401 (autouse)

pytestmark = pytest.mark.gpu
XLMR_L14, XLMR_B32, LABSE = ("multilingual-clip/XLM-Roberta-Large-Vit-L-14", "multilingual-clip/XLM-Roberta-Large-Vit-B-32",
                             "multilingual-clip/LABSE-Vit-L-14")
MODEL_FILE = Path(__file__).resolve().parent / "golden" / "unigram_golden.model"


def _text_encoder(a, sd, max_batch=8):
    from marqo_b200.engine import Encoder
    return Encoder(a["text_kind"], a, sd, max_batch=max_batch)


def _live_bytes():
    from marqo_b200 import _native as N
    n = ctypes.c_int64(0)
    N.check(N.load().b200_debug_device_bytes(ctypes.byref(n)))
    return n.value


# ------------------------------------------------------------------------------------------------------------------
# The head kernel
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("normalize", [False, True])
@pytest.mark.parametrize("w,E", [(1024, 768), (1024, 512), (768, 768)])
def test_text_head_against_fp64(gpu_required, w, E, normalize):
    """The masked mean over 1, 129 and 512 of 512 token rows, @ [w, E] + bias, against fp64; the rows past each key
    length hold large values that must not leak in."""
    from marqo_b200.engine import debug_text_head
    rng = np.random.default_rng(w + E)
    S, lens = 512, np.array([1, 129, 512], np.int32)
    x = rng.standard_normal((3, S, w)).astype(np.float32)
    for b, L in enumerate(lens):
        x[b, L:] = 1e6
    proj = (rng.standard_normal((w, E)) / np.sqrt(w)).astype(np.float32)
    bias = rng.standard_normal(E).astype(np.float32)
    pooled = np.stack([x[b, :L].astype(np.float64).mean(0) for b, L in enumerate(lens)])
    for bb in (bias, None):
        ref = pooled @ proj.astype(np.float64) + (0 if bb is None else bb.astype(np.float64))
        if normalize:
            ref /= np.linalg.norm(ref, axis=1, keepdims=True)
        got = debug_text_head(x.reshape(3 * S, w), S, lens, proj, bb, normalize=normalize)
        assert got.shape == (3, E)
        np.testing.assert_allclose(got, ref, rtol=0, atol=1e-5 * float(np.abs(ref).max()))


# ------------------------------------------------------------------------------------------------------------------
# The text towers through the C ABI
# ------------------------------------------------------------------------------------------------------------------
def _check_tower(enc, sd, a, ids, mask, sel):
    for normalize in (False, True):
        got = enc.encode_tokens(ids.numpy(), mask.numpy(), normalize=normalize)
        assert got.shape == (ids.shape[0], a["proj_dim"])
        ref = M.encode_text(sd, a, ids[sel], mask[sel], normalize)
        assert_embeddings_match(got[sel], ref, unit_norm=normalize)
        if not normalize:
            torch.testing.assert_close(torch.from_numpy(got[sel]).double().norm(dim=-1), ref.double().norm(dim=-1),
                                       rtol=1e-2, atol=0)


def test_xlmr_tower_two_layers(gpu_required):
    """XLM-R large's width at 2 layers, dimensions 512, b8 x 512 with lengths 1 to 512 and a "transformer." prefix."""
    a = M.arch(XLMR_B32, layers=2)
    sd = M.text_weights(a, seed=5)
    enc = _text_encoder(a, sd)
    try:
        g = torch.Generator().manual_seed(0)
        ids, mask = X.ragged_ids(g, 8, 512, [512, 1, 129, 40, 511, 3, 300, 2], a["vocab"])
        ids[1, 0] = 2
        ids[3, 7] = a["vocab"] - 1
        _check_tower(enc, sd, a, ids, mask, [0, 1, 2, 3])
    finally:
        enc.close()


def test_labse_full_depth_full_vocabulary(gpu_required):
    """LaBSE's 12 layers over its 501153-row word table, ids above 250002 included, b4 x 512."""
    a = M.arch(LABSE)
    sd = M.text_weights(a, seed=6)
    enc = _text_encoder(a, sd, max_batch=4)
    try:
        g = torch.Generator().manual_seed(1)
        ids = torch.randint(250003, a["vocab"], (4, 512), generator=g)
        ids[:, 0] = 101
        mask = torch.ones(4, 512, dtype=torch.int64)
        for b, L in enumerate((512, 1, 129, 60)):
            ids[b, L - 1] = 102
            ids[b, L:], mask[b, L:] = 0, 0
        ids[0, 100:200] = torch.randint(1000, 250002, (100,), generator=g)
        ids[2, 9] = a["vocab"] - 1
        _check_tower(enc, sd, a, ids, mask, [0, 1, 2, 3])
    finally:
        enc.close()


def test_513_tokens_refused_with_nothing_written(gpu_required):
    from marqo_b200._native import ERR_INVALID_ARG, NativeError
    a = M.arch(XLMR_L14, layers=1, vocab=1000)
    enc = _text_encoder(a, M.text_weights(a, seed=7), max_batch=2)
    try:
        ids = torch.full((2, 513), 5, dtype=torch.int32, device="cuda")
        out = torch.full((2, a["proj_dim"]), 7.0, device="cuda")
        torch.cuda.synchronize()
        with pytest.raises(NativeError) as e:
            enc.encode_tokens_device(ids.data_ptr(), None, 2, 513, out.data_ptr())
        assert e.value.code == ERR_INVALID_ARG
        assert bool((out == 7.0).all())
    finally:
        enc.close()


# ------------------------------------------------------------------------------------------------------------------
# Launch counts, device memory
# ------------------------------------------------------------------------------------------------------------------
def _launch_counts():
    """The M-CLIP text tower launches what the plain XLM-R tower does, with the 3-kernel projected head (2 without
    normalize) in place of bert_head's one kernel.  Each count is what the device ran (torch.profiler) in the captured
    graph's first launch.  Runs in a process of its own, as tests/test_coca_gpu.py's launch counts do."""
    from marqo_b200.engine import Encoder
    from marqo_b200.weights import random_xlmr_weights
    from test_model_launches_gpu import _kernels
    a = M.arch(XLMR_L14, layers=2, vocab=1000)
    plain = {k: v for k, v in a.items() if k not in ("kind", "proj_dim")}
    mclip, xlmr = _text_encoder(a, M.text_weights(a, 1), 4), Encoder("xlmr", plain, random_xlmr_weights(plain, 1),
                                                                     max_batch=4)
    torch.cuda.init()
    try:
        for normalize in (False, True):
            n = 3 if normalize else 2
            ids, mask = X.ragged_ids(torch.Generator().manual_seed(n), n, 40, [40, 7, 12][:n], 1000)
            ids, mask = ids.numpy(), mask.numpy()
            counts = {}
            for tag, enc in (("mclip", mclip), ("xlmr", xlmr)):
                call = lambda: enc.encode_tokens(ids, mask, normalize=normalize)
                call()
                counts[tag] = enc.last_timing()[1]
                ran = _kernels(call)
                assert len(ran) == counts[tag], f"{tag}: reported {counts[tag]}, ran {len(ran)}: {ran}"
                call()
                assert enc.last_timing()[1] == counts[tag], f"{tag}: graph replay"
            assert counts["mclip"] == counts["xlmr"] + (2 if normalize else 1), counts
    finally:
        mclip.close()
        xlmr.close()


def test_launch_counts(gpu_required):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([root, os.path.join(root, "tests"),
                                                       os.environ.get("PYTHONPATH", "")]))
    r = subprocess.run([sys.executable, "-c", "import test_multilingual_clip_gpu as t; t._launch_counts()"], cwd=root,
                       env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]


def _loader(name, seed, text_layers, **props):
    from marqo_b200 import model_registry as R
    from marqo_b200.loaders import B200MultilingualClip
    p = dict(R.get_model_properties(name), random_init=seed, max_batch=16, **props)
    p["arch"]["layers"] = text_layers
    m = B200MultilingualClip(device="cuda:0", model_properties=p)
    m.load()
    return m


def test_device_memory_returns_after_close(gpu_required):
    from _checks import WordTokenizer
    before = _live_bytes()
    m = _loader(LABSE, 3, 1, tokenizer=WordTokenizer(101, 102, 1000))
    m.encode_image([np.zeros((300, 200, 3), np.uint8)])
    m.encode_text(["w1 w2", "w3"])
    assert _live_bytes() > before
    m.close()
    assert _live_bytes() == before


# ------------------------------------------------------------------------------------------------------------------
# The image tower and the seams
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,visual", [(XLMR_B32, "ViT-B/32"), (LABSE, "ViT-L/14")])
def test_image_vectors_are_b200clips(gpu_required, name, visual):
    """The same seed gives B200Clip's image weights; the vectors are the same bits on every input path."""
    from marqo_b200 import model_registry as R
    from marqo_b200.loaders import B200Clip
    m = _loader(name, 11, 1)
    clip = B200Clip(device="cuda:0", model_properties=dict(R.get_model_properties(visual), random_init=11, max_batch=16))
    clip.load()
    try:
        rng = np.random.default_rng(2)
        images = [rng.integers(0, 256, (int(h), int(w), 3), dtype=np.uint8)
                  for h, w in zip(rng.integers(150, 500, 6), rng.integers(150, 500, 6))]
        for normalize in (True, False):
            np.testing.assert_array_equal(m.encode_image(images, normalize=normalize),
                                          clip.encode_image(images, normalize=normalize))
        dev = [torch.from_numpy(a).cuda() for a in images[:3]]
        np.testing.assert_array_equal(m.encode(dev, default="image"), clip.encode(dev, default="image"))
        np.testing.assert_array_equal(m.encode_to_device(images, default="image").cpu().numpy(),
                                      clip.encode_to_device(images, default="image").cpu().numpy())
    finally:
        m.close()
        clip.close()


def test_vectorise_into_index_and_search(gpu_required, score_oracle, monkeypatch):
    """vectorise of texts (the C++ Unigram tokenizer) and images -> GpuTensorIndex -> search: the text vectors against
    the M-CLIP oracle on the same seeded weights, the hits against the score oracle; a text over 512 tokens is refused.
    Marqo declares 5 GB for this name (the multilingual_clip type), over its default 4 GB device threshold."""
    import sentencepiece as spm
    from marqo_b200 import model_registry as R, s2_inference as s2
    from marqo_b200.errors import VectoriseError
    from marqo_b200.s2_inference import Modality
    monkeypatch.setenv("MARQO_MAX_CUDA_MODEL_MEMORY", "16")
    s2.clear_loaded_models()
    name = XLMR_B32
    props = dict(R.get_model_properties(name), random_init=31, max_batch=32, vocab_file=str(MODEL_FILE))
    props["arch"]["layers"] = 2
    rng = np.random.default_rng(8)
    images = [rng.integers(0, 256, (int(h), int(w), 3), dtype=np.uint8)
              for h, w in zip(rng.integers(150, 400, 20), rng.integers(150, 400, 20))]
    alphabet = "abcdefghijklmnopqrstuvwxyzéñü東京大学日本語абвгдежзαβγ "
    texts = ["".join(alphabet[int(x)] for x in rng.integers(0, len(alphabet), size=n)) for n in rng.integers(1, 80, 20)]
    kw = dict(model_properties=props, device="cuda:0", normalize_embeddings=True)
    image_docs = np.asarray(s2.vectorise(name, images, modality=Modality.IMAGE, **kw), np.float32)
    text_docs = np.asarray(s2.vectorise(name, texts, **kw), np.float32)
    queries = ["東京 大学", "привет мир", "café", "αβγ"]
    q = np.asarray(s2.vectorise(name, queries, **kw), np.float32)
    with pytest.raises(VectoriseError):
        s2.vectorise(name, ["a " * 600], **kw)
    s2.clear_loaded_models()
    assert image_docs.shape == (20, 512) and text_docs.shape == (20, 512)

    sp = spm.SentencePieceProcessor(model_file=str(MODEL_FILE))
    a = props["arch"]
    sd = M.text_weights(a, 32)   # random_init + 1: the loader's text seed

    def oracle(batch):
        rows = [X.fairseq_ids(sp, t) for t in batch]
        L = max(len(r) for r in rows)
        ids = torch.tensor([r + [1] * (L - len(r)) for r in rows])
        mask = torch.tensor([[1] * len(r) + [0] * (L - len(r)) for r in rows])
        return M.encode_text(sd, a, ids, mask)

    assert_embeddings_match(q, oracle(queries))
    assert_embeddings_match(text_docs[:4], oracle(texts[:4]))
    assert_index_search_matches(score_oracle, np.concatenate([image_docs, text_docs]), np.concatenate([q, image_docs[:2]]))
