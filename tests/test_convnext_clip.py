"""ConvNeXt CLIP on the CPU: the registry entries against the reference's, the fp32 oracle (tests/_convnext_oracle.py)
against transformers.ConvNextModel on the same weights, and the checkpoint names random_clip_convnext_weights
produces."""
import numpy as np
import pytest
import torch

import _convnext_oracle as O

# model_registry.py:274-343 of the reference: name -> dimensions
REFERENCE = {
    "open_clip/convnext_base/laion400m_s13b_b51k": 512,
    "open_clip/convnext_base_w/laion2b_s13b_b82k": 640,
    "open_clip/convnext_base_w/laion2b_s13b_b82k_augreg": 640,
    "open_clip/convnext_base_w/laion_aesthetic_s13b_b82k": 640,
    "open_clip/convnext_base_w_320/laion_aesthetic_s13b_b82k": 640,
    "open_clip/convnext_base_w_320/laion_aesthetic_s13b_b82k_augreg": 640,
    "open_clip/convnext_large_d/laion2b_s26b_b102k_augreg": 768,
    "open_clip/convnext_large_d_320/laion2b_s29b_b131k_ft": 768,
    "open_clip/convnext_large_d_320/laion2b_s29b_b131k_ft_soup": 768,
    "open_clip/convnext_xxlarge/laion2b_s34b_b82k_augreg": 1024,
    "open_clip/convnext_xxlarge/laion2b_s34b_b82k_augreg_rewind": 1024,
    "open_clip/convnext_xxlarge/laion2b_s34b_b82k_augreg_soup": 1024,
}


def test_registry_entries():
    from marqo_b200 import model_registry as R
    assert set(R.CONVNEXT_MODELS) == set(REFERENCE)
    for name, dims in REFERENCE.items():
        e = R.find_model(name)
        assert e is R.CONVNEXT_MODELS[name] and name not in R.all_models()
        a = e["arch"]
        assert e["dimensions"] == dims == a["embed_dim"]
        assert e["pretrained"] == name.split("/")[2] and e["type"] == R.TYPE_OPEN_CLIP
        assert a["kind"] == "clip_convnext" and "vision" not in a
        assert a["mlp"] == 4 * a["width"] and a["width"] == 64 * a["heads"] and a["ctx"] == 77
        assert (a["convnext"]["head"] == "mlp") == ("large_d" in name)
        assert a["convnext"]["ln_eps"] == (1e-5 if "xxlarge" in name else 1e-6)
        assert R.get_model_properties(name)["dimensions"] == dims


def test_convnext_names_are_in_no_other_table():
    from marqo_b200 import model_registry as R
    others = [R.MODELS, R.MPNET_MODELS, R.SIGLIP_MODELS, R.XLMR_MODELS, R.RESNET_MODELS]
    assert not any(set(R.CONVNEXT_MODELS) & set(t) for t in others)
    assert not any("convnext" in n for t in others for n in t)


def _cx(dims, depths, eps=1e-6, head="linear", image=64):
    return {"dims": dims, "depths": depths, "image_size": image, "ln_eps": eps, "head": head}


# the base, large and xxlarge stage widths at reduced depth and small images
TRUNKS = [([128, 256, 512, 1024], [1, 1, 2, 1], 64), ([192, 384, 768, 1536], [2, 1, 1, 1], 96),
          ([384, 768, 1536, 3072], [1, 2, 1, 1], 64)]


@pytest.mark.parametrize("dims,depths,S", TRUNKS)
def test_oracle_trunk_matches_transformers_convnext(dims, depths, S):
    from transformers import ConvNextConfig, ConvNextModel
    from marqo_b200.weights import random_clip_convnext_weights
    cx = _cx(dims, depths, image=S)
    arch = {"embed_dim": 64, "layers": 0, "convnext": cx}
    sd = {k: torch.from_numpy(v) for k, v in random_clip_convnext_weights(arch, seed=sum(depths)).items()}
    cfg = ConvNextConfig(num_channels=3, patch_size=4, num_stages=4, hidden_sizes=dims, depths=depths,
                         hidden_act="gelu", layer_norm_eps=1e-6, layer_scale_init_value=1e-6, drop_path_rate=0.0,
                         image_size=S)
    hf = ConvNextModel(cfg).eval()
    missing, unexpected = hf.load_state_dict(O.to_hf(sd), strict=False)
    assert not missing and not unexpected
    x = torch.randn(2, 3, S, S, generator=torch.Generator().manual_seed(S))
    with torch.no_grad():
        ref = hf(x).pooler_output
        got = O.pooled({k: v.float() for k, v in sd.items()}, cx, x)
    torch.testing.assert_close(got, ref, rtol=1e-4, atol=1e-4)


def _expected_shapes(arch):
    """The parameters b200_model_finalize reads for a clip_convnext arch, by name."""
    cx, E = arch["convnext"], arch["embed_dim"]
    dims, t = cx["dims"], "visual.trunk."
    s = {t + "stem.0.weight": (dims[0], 3, 4, 4), t + "stem.0.bias": (dims[0],), t + "stem.1.weight": (dims[0],),
         t + "stem.1.bias": (dims[0],), t + "head.norm.weight": (dims[3],), t + "head.norm.bias": (dims[3],)}
    for st, (C, depth) in enumerate(zip(dims, cx["depths"])):
        p = f"{t}stages.{st}."
        if st:
            s.update({p + "downsample.0.weight": (dims[st - 1],), p + "downsample.0.bias": (dims[st - 1],),
                      p + "downsample.1.weight": (C, dims[st - 1], 2, 2), p + "downsample.1.bias": (C,)})
        for i in range(depth):
            b = f"{p}blocks.{i}."
            s.update({b + "conv_dw.weight": (C, 1, 7, 7), b + "conv_dw.bias": (C,), b + "norm.weight": (C,),
                      b + "norm.bias": (C,), b + "mlp.fc1.weight": (4 * C, C), b + "mlp.fc1.bias": (4 * C,),
                      b + "mlp.fc2.weight": (C, 4 * C), b + "mlp.fc2.bias": (C,), b + "gamma": (C,)})
    if cx["head"] == "mlp":
        s.update({"visual.head.mlp.fc1.weight": (2 * E, dims[3]), "visual.head.mlp.fc1.bias": (2 * E,),
                  "visual.head.mlp.fc2.weight": (E, 2 * E)})
    else:
        s["visual.head.proj.weight"] = (E, dims[3])
    return s


@pytest.mark.parametrize("name", ["open_clip/convnext_base_w/laion2b_s13b_b82k",
                                  "open_clip/convnext_large_d/laion2b_s26b_b102k_augreg"])
def test_random_weights_carry_the_names_finalize_requires(name):
    from marqo_b200 import model_registry as R
    from marqo_b200.weights import random_clip_convnext_weights, random_clip_weights
    arch = R.get_model_properties(name)["arch"]
    arch["convnext"]["depths"] = [1, 1, 2, 1]   # the names do not depend on the depth beyond the loop
    sd = random_clip_convnext_weights(arch, seed=3)
    text = {k: v.shape for k, v in random_clip_weights(
        {"embed_dim": arch["embed_dim"], "text": {k: arch[k] for k in ("width", "layers", "heads", "mlp", "ctx", "vocab")}},
        seed=4).items()}
    want = {**_expected_shapes(arch), **text}
    assert {k: v.shape for k, v in sd.items()} == want
    assert all(v.dtype == np.float32 for v in sd.values())


class _FakeLoader:
    seen = []

    def __init__(self, device, model_properties, **kwargs):
        self.model_properties = model_properties
        _FakeLoader.seen.append(model_properties)

    def load(self):
        pass

    def encode(self, content, normalize=True, **kwargs):
        n = len(content) if isinstance(content, list) else 1
        return np.ones((n, self.model_properties["dimensions"]), np.float32)


@pytest.mark.parametrize("name,dims", [("open_clip/convnext_base_w/laion2b_s13b_b82k", 640),
                                       ("open_clip/convnext_large_d_320/laion2b_s29b_b131k_ft", 768)])
def test_vectorise_routes_convnext_to_the_open_clip_loader(monkeypatch, name, dims):
    from marqo_b200 import loaders, model_registry as R, s2_inference
    monkeypatch.setitem(loaders.LOADERS, R.TYPE_OPEN_CLIP, _FakeLoader)
    monkeypatch.setattr(s2_inference, "_available_models", {})
    _FakeLoader.seen.clear()
    out = s2_inference.vectorise(name, "a photo of a dog", device="cuda:0")
    assert len(out) == 1 and len(out[0]) == dims
    (props,) = _FakeLoader.seen
    assert props["type"] == R.TYPE_OPEN_CLIP and props["arch"]["kind"] == "clip_convnext"


def test_clip_tokenizer_takes_ctx_from_the_top_level(tmp_path):
    from marqo_b200 import model_registry as R
    from marqo_b200.loaders import B200OpenCLIP
    import marqo_b200.tokenizers as T
    seen = {}

    class Fake:
        def __init__(self, path, context_length):
            seen["ctx"] = context_length

    m = B200OpenCLIP(device="cuda:0", model_properties={"merges_file": "unused"})
    m.arch = R.get_model_properties("open_clip/convnext_xxlarge/laion2b_s34b_b82k_augreg")["arch"]
    orig = T.ClipBpeTokenizer
    T.ClipBpeTokenizer = Fake
    try:
        m._default_tokenizer()
    finally:
        T.ClipBpeTokenizer = orig
    assert seen["ctx"] == 77
