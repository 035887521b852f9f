"""Every device buffer the library allocates is released again.  Each scenario reads the library's own count of live
device bytes (b200_debug_device_bytes) before and after, and the difference must come back to zero: index life cycles
with every growth path, calls rejected after they allocated, the exchange buffer, an encoder (also one whose finalize
fails), one encoder of each of the EVA02, big-ViT, ConvNeXt and GTE kinds through its encode calls, the JPEG decoder
and the resize temporaries.  cudaMemGetInfo is not used: other processes share the card."""
import contextlib
import ctypes as C
import gc
import io

import numpy as np
import pytest
import torch

import _big_vit_oracle as B
import _eva02_oracle as V
import _gte_oracle as G
from _checks import clip_text_ids
from marqo_b200 import _native as N

pytestmark = pytest.mark.gpu
DIM = 64


def _live_bytes() -> int:
    n = C.c_int64(0)
    N.check(N.load().b200_debug_device_bytes(C.byref(n)))
    return n.value


@contextlib.contextmanager
def _released():
    before = _live_bytes()
    yield before
    gc.collect()
    assert _live_bytes() == before


def _vecs(rng, m):
    return rng.standard_normal((m, DIM)).astype(np.float32)


def _raises(code, fn, *args, **kwargs):
    with pytest.raises(N.NativeError) as e:
        fn(*args, **kwargs)
    assert e.value.code == code, e.value


@pytest.mark.parametrize("metric", ["prenormalized-angular", "euclidean"])
def test_index_life_cycle(gpu_required, tmp_path, metric):
    from marqo_b200.engine import RowStore
    rng = np.random.default_rng(0)
    with _released() as before:
        ix = RowStore(DIM, metric=metric, capacity=0)
        assert _live_bytes() > before
        # grow from the minimum capacity over several adds: host and device, with and without document ids
        ix.add(_vecs(rng, 100))
        ix.add(_vecs(rng, 300), doc_ids=np.arange(100, 400))
        d_v = torch.from_numpy(_vecs(rng, 500)).cuda()
        d_ids = torch.arange(400, 900, dtype=torch.int32, device="cuda")
        ix.add_device(d_v.data_ptr(), 500, d_ids.data_ptr())
        ix.add_device(d_v.data_ptr(), 500)
        ix.add_device_docs(d_v.data_ptr(), np.arange(1400, 1900))
        torch.cuda.synchronize()
        assert len(ix) == 1900
        ix.delete_rows(np.arange(0, 1900, 7))
        ix.compact()
        # attribute columns: set, then grown past their capacity twice
        ix.set_attributes(0, np.arange(0, 500), rng.random(500))
        ix.set_attributes_multi([1, 2, 3], [10, 1500, 3000], [1.0, 2.0, 3.0])
        ix.set_attributes(4, [6000], [0.5])
        ix.set_attributes(-1, [10], None)
        n_docs = 1900
        bits = np.full((n_docs + 31) // 32, 0xFFFFFFFF, dtype=np.uint32)
        bits[::3] = 0
        doc, _, _ = ix.search(_vecs(rng, 3), 10, mult=[(0, 1.5)], add=[(1, 0.25)], filter_bits=bits,
                              filter_docs=n_docs, filter_tag=7)
        assert (doc >= 0).all()
        path = tmp_path / "ix.b200"
        ix.save(str(path))
        loaded = RowStore.load(str(path))
        assert len(loaded) == len(ix)
        loaded.close()
        ix.close()


def test_deep_search_scratch(gpu_required):
    """k = 5000 over 7000 documents collects more rows than the device finalize holds (FIN_CAP = 4096): the collect
    buffer grows once, and the host finalize's per-call scratch is released by every call."""
    from marqo_b200.engine import RowStore
    rng = np.random.default_rng(1)
    with _released():
        ix = RowStore(DIM, capacity=0)
        ix.add(_vecs(rng, 7000))
        q = _vecs(rng, 2)
        doc, _, _ = ix.search(q, 5000)
        assert (doc >= 0).all() and len(np.unique(doc[0])) == 5000
        after_first = _live_bytes()
        ix.search(q, 5000)
        assert _live_bytes() == after_first
        ix.close()


def test_rejected_add_after_growth(gpu_required):
    from marqo_b200.engine import RowStore
    rng = np.random.default_rng(2)
    with _released():
        ix = RowStore(DIM, capacity=0)
        ix.add(_vecs(rng, 50))
        bad = _vecs(rng, 1000)   # grows the corpus before the values are checked
        bad[700, 3] = np.nan
        _raises(N.ERR_INVALID_ARG, ix.add, bad)
        assert len(ix) == 50
        ix.close()


def test_truncated_snapshot(gpu_required, tmp_path):
    from marqo_b200.engine import RowStore
    rng = np.random.default_rng(3)
    path, cut = tmp_path / "full.b200", tmp_path / "cut.b200"
    with _released():
        ix = RowStore(DIM, capacity=0)
        ix.add(_vecs(rng, 600))
        ix.set_attributes(0, np.arange(600), rng.random(600))
        ix.save(str(path))
        ix.close()
    data = path.read_bytes()
    with _released():
        for size in (len(data) // 2, len(data) - 100):
            with open(cut, "wb") as f:
                f.write(data[:size])
            _raises(N.ERR_INVALID_ARG, RowStore.load, str(cut))


def test_rejected_negative_multiplier(gpu_required):
    from marqo_b200.engine import RowStore
    rng = np.random.default_rng(4)
    with _released():
        ix = RowStore(DIM, capacity=0)
        ix.add(_vecs(rng, 400), doc_ids=np.repeat(np.arange(200), 2))   # two chunks per document
        ix.set_attributes(0, np.arange(200), rng.random(200) + 0.5)
        _raises(N.ERR_UNSUPPORTED, ix.search, _vecs(rng, 2), 10, mult=[(0, -1.0)])
        ix.close()


def test_exchange_single_rank(gpu_required):
    from marqo_b200.engine import Exchange
    with _released() as before:
        ex = Exchange(0, 0, 1)
        assert _live_bytes() > before
        ex.open([ex.handle])
        ex.close()


def _small_bert():
    """hf/all-MiniLM-L6-v2's arch with two layers and a short vocabulary."""
    from marqo_b200.model_registry import MODELS
    from oracle import encoders as E
    arch = dict(MODELS["hf/all-MiniLM-L6-v2"]["arch"], layers=2, vocab=1000, max_pos=64)
    cfg = E.BertCfg(arch["width"], arch["layers"], arch["heads"], arch["mlp"], vocab=arch["vocab"],
                    max_pos=arch["max_pos"], type_vocab=arch["type_vocab"], pool=arch["pool"])
    return arch, E.make_bert_weights(cfg, seed=5)


def test_encoder_life_cycle(gpu_required):
    from marqo_b200.engine import Encoder
    arch, sd = _small_bert()
    ids = np.random.default_rng(5).integers(0, arch["vocab"], size=(4, 16)).astype(np.int32)
    with _released() as before:
        enc = Encoder("bert", arch, sd, max_batch=8)
        assert _live_bytes() > before
        for _ in range(3):   # eager, captured into a CUDA graph, replayed
            out = enc.encode_tokens(ids)
        assert out.shape == (4, arch["width"]) and np.isfinite(out).all()
        enc.close()


def _convnext_arch():
    from marqo_b200 import model_registry as R
    a = R.get_model_properties("open_clip/convnext_base_w/laion2b_s13b_b82k")["arch"]
    a["convnext"]["depths"], a["layers"] = [1, 1, 1, 1], 0
    return a


def _photos(enc):
    enc.encode_images_u8(np.zeros((2, 300, 200, 3), np.uint8))


def _clip_text(enc):
    enc.encode_tokens(clip_text_ids(2, 1).numpy())


def _gte_ragged(enc):
    ids, mask = G.ragged_ids(torch.Generator().manual_seed(3), [200, 5], 200, G.STELLA.vocab)
    enc.encode_tokens(ids.numpy(), mask.numpy())


# kind, arch (one layer per tower), the encode calls; seeded weights, max_batch 8
_TOWERS = {
    "eva02": ("clip_eva", lambda: V.arch(V.L14, eva_layers=1, text_layers=1), (_photos, _clip_text)),
    "big_vit": ("clip", lambda: B.arch(B.BIG_G, vision_layers=1, text_layers=1), (_photos, _clip_text)),
    "convnext": ("clip_convnext", _convnext_arch,
                 (lambda enc: enc.encode_images_u8(np.zeros((2, 256, 256, 3), np.uint8)),)),
    "gte": ("gte", lambda: G.engine_config(G.GteCfg(layers=1)), (_gte_ragged,)),
}


@pytest.mark.parametrize("tower", list(_TOWERS))
def test_tower_kind_life_cycle(gpu_required, tower):
    from marqo_b200.engine import Encoder
    from marqo_b200.weights import random_weights
    kind, arch, calls = _TOWERS[tower]
    arch = arch()
    sd = random_weights(kind, arch, 9)
    with _released() as before:
        enc = Encoder(kind, arch, sd, max_batch=8)
        assert _live_bytes() > before
        for call in calls:
            call(enc)
        enc.close()


def test_encoder_failed_finalize(gpu_required):
    from marqo_b200.engine import Encoder
    arch, sd = _small_bert()
    del sd["encoder.layer.1.output.LayerNorm.bias"]   # read last: layer 0 and part of layer 1 are already converted
    with _released():
        _raises(N.ERR_MISSING_WEIGHT, Encoder, "bert", arch, sd, max_batch=8)


def test_jpeg_decode_and_resize(gpu_required):
    from PIL import Image
    from marqo_b200.engine import debug_resize
    from marqo_b200.image_decode import decode_jpegs_to_device
    rng = np.random.default_rng(6)
    buf = io.BytesIO()
    Image.fromarray(rng.integers(0, 256, size=(48, 80, 3), dtype=np.uint8)).save(buf, format="JPEG", quality=85)
    jpeg = buf.getvalue()
    with _released():
        out = decode_jpegs_to_device([jpeg, jpeg], device=0)
        want = np.asarray(Image.open(io.BytesIO(jpeg)).convert("RGB"))
        assert all(np.array_equal(t.cpu().numpy(), want) for t in out)
        del out
        resized = debug_resize(rng.integers(0, 256, size=(2, 40, 70, 3), dtype=np.uint8), 32)
        assert resized.shape == (2, 32, 32, 3)
