"""The `multilingual_clip` loader type on the CPU: the registry entries and their declared sizes against the
reference's own (tests/golden/multilingual_clip_golden.json, written by tests/golden/make_multilingual_clip_golden.py),
the registry walks of the shape tests left as they were, the M-CLIP text oracle against transformers, and the loader's
routing and refusals."""
import json
from pathlib import Path

import numpy as np
import pytest
import torch

import _mclip_oracle as M

GOLDEN = json.loads((Path(__file__).resolve().parent / "golden" / "multilingual_clip_golden.json").read_text())
UNSERVED = "multilingual-clip/XLM-R Large Vit-B/16+"
SERVED = sorted(n for n in GOLDEN if n != UNSERVED)
XLMR_L14, XLMR_B32, LABSE = ("multilingual-clip/XLM-Roberta-Large-Vit-L-14", "multilingual-clip/XLM-Roberta-Large-Vit-B-32",
                             "multilingual-clip/LABSE-Vit-L-14")


@pytest.mark.parametrize("name", SERVED)
def test_registry_entries_match_the_reference(name):
    from marqo_b200 import model_registry as R, s2_inference as s2
    e = R.get_model_properties(name)
    table = R.MULTILINGUAL_CLIP_MODELS
    assert R.find_model(name) is table[name] and R.all_models()[name] is table[name]
    assert R.served_models()[name] is table[name]
    ref = dict(GOLDEN[name]["properties"], type=R.TYPE_MULTILINGUAL_CLIP)
    assert {k: v for k, v in e.items() if k != "arch"} == ref
    assert s2.get_model_size(name, e) == GOLDEN[name]["model_size"]
    a = e["arch"]
    assert a["kind"] == "mclip" and a["proj_dim"] == e["dimensions"]
    assert "openai/" + a["visual"] == e["visual_model"] and a["visual"] in R.OPENAI_CLIP_MODELS


def test_text_tower_shapes():
    from marqo_b200 import model_registry as R
    for name in (XLMR_L14, XLMR_B32):
        a = R.MULTILINGUAL_CLIP_MODELS[name]["arch"]
        assert a["text_kind"] == "xlmr"
        assert {k: a[k] for k in ("width", "layers", "heads", "mlp", "vocab", "max_pos", "pad_id", "ln_eps")} == dict(
            width=1024, layers=24, heads=16, mlp=4096, vocab=250002, max_pos=514, pad_id=1, ln_eps=1e-5)
    a = R.MULTILINGUAL_CLIP_MODELS[LABSE]["arch"]
    assert a["text_kind"] == "bert"
    assert {k: a[k] for k in ("width", "layers", "heads", "mlp", "vocab", "max_pos", "type_vocab", "ln_eps")} == dict(
        width=768, layers=12, heads=12, mlp=3072, vocab=501153, max_pos=512, type_vocab=2, ln_eps=1e-12)


def test_vit_b_16_plus_stays_unserved():
    from marqo_b200 import model_registry as R, s2_inference as s2
    from marqo_b200.errors import InvalidModelPropertiesError, UnknownModelError
    assert R.find_model(UNSERVED) is None and UNSERVED not in R.served_models()
    with pytest.raises(UnknownModelError):
        s2.validate_model_properties(UNSERVED, None)
    with pytest.raises(InvalidModelPropertiesError, match="not served"):
        s2.validate_model_properties(UNSERVED, dict(GOLDEN[UNSERVED]["properties"]))


def test_registry_walks_see_no_new_shapes(monkeypatch):
    """The GEMM widths, layer variants, patch embeddings and resize sizes the shape tests walk the registry for are the
    same with and without MULTILINGUAL_CLIP_MODELS."""
    from marqo_b200 import model_registry as R
    from _checks import served_resize_sizes
    from test_gemm_shapes_gpu import _served_layers
    from test_layers_gpu import _variants
    from test_patch_embed_gpu import _served_patch_embeddings

    def walks():
        return (_served_layers(), sorted(_variants()), _served_patch_embeddings()[0],
                served_resize_sizes("crop"), served_resize_sizes("squash"))

    with_mclip = walks()
    assert {w for w, _ in with_mclip[0]} == {384, 512, 768, 1024}
    assert not _served_patch_embeddings()[1]
    monkeypatch.setattr(R, "MULTILINGUAL_CLIP_MODELS", {})
    assert walks() == with_mclip


@pytest.mark.parametrize("name", [XLMR_B32, LABSE])
def test_oracle_against_transformers(name):
    """The M-CLIP oracle at 2 layers with seeded weights against transformers' XLMRobertaModel / BertModel and a torch
    Linear: right-padded rows of lengths 1 to 40, and ids near the top of the vocabulary."""
    a = M.arch(name, layers=2, vocab=1000)
    sd = M.text_weights(a, seed=3)
    g = torch.Generator().manual_seed(1)
    pad = a["pad_id"]
    ids = torch.randint(4, a["vocab"], (5, 40), generator=g)
    mask = torch.ones(5, 40, dtype=torch.int64)
    for b, L in enumerate((40, 1, 17, 2, 33)):
        ids[b, L:], mask[b, L:] = pad, 0
    ids[2, 5] = a["vocab"] - 1
    want = M.hf_encode_text(sd, a, ids, mask)
    got = M.encode_text(sd, a, ids, mask, normalize=False)
    assert got.shape == (5, a["proj_dim"])
    torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-4)
    unit = M.encode_text(sd, a, ids, mask)
    torch.testing.assert_close(unit, want / want.norm(dim=-1, keepdim=True), rtol=1e-4, atol=1e-5)


# ------------------------------------------------------------------------------------------------------------------
# Routing and refusals
# ------------------------------------------------------------------------------------------------------------------
def test_routing():
    from marqo_b200 import loaders, model_registry as R, s2_inference as s2
    props = s2.validate_model_properties(LABSE, None)
    assert loaders.get_model_loader(LABSE, props) is loaders.B200MultilingualClip
    explicit = s2.validate_model_properties(XLMR_B32, {"type": "multilingual_clip", "dimensions": 512})
    assert explicit["type"] == R.TYPE_MULTILINGUAL_CLIP and explicit["arch"] == R.MULTILINGUAL_CLIP_MODELS[XLMR_B32]["arch"]
    assert not s2.is_preprocess_image_model(props)   # PREPROCESS_IMAGE_MODEL_LIST is [clip, open_clip]


@pytest.mark.parametrize("device", [None, ""])
def test_missing_device_is_an_internal_error(device):
    from marqo_b200.errors import InternalError
    from marqo_b200.loaders import B200MultilingualClip
    with pytest.raises(InternalError, match="`device` is required for loading MULTILINGUAL CLIP models!"):
        B200MultilingualClip(device=device, model_properties={"type": "multilingual_clip"})


@pytest.mark.parametrize("missing", ["visual_weights", "textual_weights"])
def test_weights_are_required(missing):
    from marqo_b200 import model_registry as R
    from marqo_b200.errors import ModelLoadError
    from marqo_b200.loaders import B200MultilingualClip
    props = dict(R.get_model_properties(XLMR_B32), visual_weights={}, textual_weights={})
    del props[missing]
    with pytest.raises(ModelLoadError, match=missing):
        B200MultilingualClip(device="cuda:0", model_properties=props).load()


class _FakeEncoder:
    """Records encode_tokens calls in place of the GPU text Encoder."""
    embed_dim = 4

    def __init__(self):
        self.calls = []

    def encode_tokens(self, ids, mask, normalize=True):
        self.calls.append((ids, mask, normalize))
        return np.zeros((ids.shape[0], self.embed_dim), np.float32)


def _loaded(max_tokens=512):
    from _checks import WordTokenizer
    from marqo_b200 import model_registry as R
    from marqo_b200.loaders import B200MultilingualClip
    m = B200MultilingualClip(device="cuda:0", model_properties=R.get_model_properties(XLMR_B32))
    m.text_model, m.max_tokens = _FakeEncoder(), max_tokens
    m.tokenizer = WordTokenizer(0, 2, 4)
    return m


def test_text_pads_to_the_longest_and_routes_to_the_text_encoder():
    m = _loaded()
    out = m.encode(["w1 w2 w3", "w5"], normalize=False)
    assert out.shape == (2, 4)
    ids, mask, normalize = m.text_model.calls[0]
    np.testing.assert_array_equal(ids, [[0, 5, 6, 7, 2], [0, 9, 2, 0, 0]])
    np.testing.assert_array_equal(mask, [[1, 1, 1, 1, 1], [1, 1, 1, 0, 0]])
    assert ids.dtype == np.int32 and mask.dtype == np.int32 and normalize is False
    m.encode_text("w1")
    assert m.text_model.calls[1][0].shape == (1, 3) and m.text_model.calls[1][2] is True


def test_text_over_the_limit_is_refused_not_truncated():
    from marqo_b200.errors import VectoriseError
    m = _loaded()
    m.encode_text([" ".join(["w1"] * 510)])   # 512 tokens with <s> and </s>
    with pytest.raises(VectoriseError, match="longer than the 512 tokens"):
        m.encode_text(["w1", " ".join(["w1"] * 511)])
    assert len(m.text_model.calls) == 1
