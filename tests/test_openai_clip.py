"""The `clip` and `fp16_clip` loader types on the CPU: the registry entries against the reference's own
(tests/golden/clip_registry_golden.json, written by tests/golden/make_clip_registry_golden.py), their declared sizes,
the routing of vectorise to B200Clip / B200Fp16Clip, the loaders' refusals, the arch read from an OpenAI-format
state dict's shapes, TorchScript checkpoints, and the ResNet oracle at the wide ResNets' widths."""
import json
from pathlib import Path

import numpy as np
import pytest
import torch

import _resnet_oracle as O

GOLDEN = json.loads((Path(__file__).resolve().parent / "golden" / "clip_registry_golden.json").read_text())
# the reference's name -> the open_clip entry of the same network (same checkpoint, QuickGELU, same preprocessing)
TWINS = {"ViT-B/32": "open_clip/ViT-B-32/openai", "ViT-B/16": "open_clip/ViT-B-16/openai",
         "ViT-L/14": "open_clip/ViT-L-14/openai", "RN50": "open_clip/RN50/openai", "RN101": "open_clip/RN101/openai"}
# RN50x4, RN50x16 and RN50x64 run through custom checkpoints; their names are not registered (module docstring of
# model_registry)
WIDE = ("RN50x4", "RN50x16", "RN50x64")
SERVED = sorted(n for n in GOLDEN if n not in WIDE)


def _type(ref_type):
    from marqo_b200 import model_registry as R
    return {"clip": R.TYPE_CLIP, "fp16_clip": R.TYPE_FP16_CLIP}[ref_type]


@pytest.mark.parametrize("name", SERVED)
def test_registry_entries_match_the_reference(name):
    from marqo_b200 import model_registry as R, s2_inference as s2
    e = R.get_model_properties(name)
    assert R.find_model(name) is R.OPENAI_CLIP_MODELS[name]
    assert R.all_models()[name] is R.OPENAI_CLIP_MODELS[name] and R.served_models()[name] is R.OPENAI_CLIP_MODELS[name]
    ref = dict(GOLDEN[name]["properties"], type=_type(GOLDEN[name]["properties"]["type"]))
    assert {k: v for k, v in e.items() if k != "arch"} == ref
    assert s2.get_model_size(name, e) == GOLDEN[name]["model_size"]
    assert e["arch"]["act"] == "quickgelu" and e["arch"]["embed_dim"] == e["dimensions"]


def test_wide_resnet_names_stay_unregistered():
    from marqo_b200 import model_registry as R
    assert set(R.OPENAI_CLIP_MODELS) == set(SERVED)
    for name in WIDE:
        assert R.find_model(name) is None and name not in R.served_models()
        assert R.WIDE_RESNET_ARCHS[name]["embed_dim"] == GOLDEN[name]["properties"]["dimensions"]


@pytest.mark.parametrize("name", sorted(TWINS))
def test_arch_is_the_open_clip_twins(name):
    from marqo_b200 import model_registry as R
    assert R.get_model_properties(name)["arch"] == R.get_model_properties(TWINS[name])["arch"]
    if name.startswith("ViT"):
        assert R.get_model_properties("fp16/" + name)["arch"] == R.get_model_properties(name)["arch"]


def test_wide_arches():
    from marqo_b200 import model_registry as R
    x16, x64 = R.WIDE_RESNET_ARCHS["RN50x16"], R.WIDE_RESNET_ARCHS["RN50x64"]
    assert x16["resnet"] == {"layers": [6, 8, 18, 8], "width": 96, "heads": 48, "image_size": 384}
    assert (x16["embed_dim"], x16["width"], x16["heads"], x16["layers"], x16["mlp"]) == (768, 768, 12, 12, 3072)
    assert x64["resnet"] == {"layers": [3, 15, 36, 10], "width": 128, "heads": 64, "image_size": 448}
    assert (x64["embed_dim"], x64["width"], x64["heads"], x64["layers"], x64["mlp"]) == (1024, 1024, 16, 12, 4096)
    v336 = R.get_model_properties("ViT-L/14@336px")["arch"]
    assert v336["vision"] == dict(R.get_model_properties("ViT-L/14")["arch"]["vision"], image_size=336)


# ------------------------------------------------------------------------------------------------------------------
# Routing and the loaders' own behaviour
# ------------------------------------------------------------------------------------------------------------------
class _FakeLoader:
    seen = []

    def __init__(self, device=None, model_properties=None, model_auth=None):
        self.model_properties = model_properties
        _FakeLoader.seen.append(model_properties)

    def load(self):
        pass

    def encode(self, content, normalize=True, **kwargs):
        n = len(content) if isinstance(content, list) else 1
        return np.ones((n, self.model_properties["dimensions"]), np.float32)


@pytest.mark.parametrize("name,props", [("ViT-B/32", None), ("ViT-L/14@336px", None), ("fp16/ViT-L/14", None),
                                        ("my-clip", {"type": "clip", "dimensions": 640, "localpath": "/x/RN50x4.pt"}),
                                        ("my-b32", {"type": "clip", "dimensions": 512, "name": "ViT-B/32"})])
def test_vectorise_routes_to_the_clip_loaders(monkeypatch, name, props):
    from marqo_b200 import loaders, model_registry as R, s2_inference
    assert loaders.LOADERS[R.TYPE_CLIP] is loaders.B200Clip
    assert loaders.LOADERS[R.TYPE_FP16_CLIP] is loaders.B200Fp16Clip
    for t in (R.TYPE_CLIP, R.TYPE_FP16_CLIP):
        monkeypatch.setitem(loaders.LOADERS, t, _FakeLoader)
    monkeypatch.setattr(s2_inference, "_available_models", {})
    _FakeLoader.seen.clear()
    out = s2_inference.vectorise(name, "a photo of a dog", model_properties=props, device="cuda:0")
    (seen,) = _FakeLoader.seen
    assert len(out) == 1 and len(out[0]) == seen["dimensions"]
    assert seen["type"] == (R.TYPE_FP16_CLIP if name.startswith("fp16/") else R.TYPE_CLIP)
    if props is not None and "localpath" in props:
        assert "arch" not in seen   # read from the checkpoint by the loader
    else:
        assert seen["arch"] == R.get_model_properties(props["name"] if props else name)["arch"]


def test_unknown_types_still_refused():
    from marqo_b200 import s2_inference
    from marqo_b200.errors import InvalidModelPropertiesError
    with pytest.raises(InvalidModelPropertiesError, match="not served"):
        s2_inference.validate_model_properties("x", {"type": "multilingual_clip", "dimensions": 768})


@pytest.mark.parametrize("cls", ["B200Clip", "B200Fp16Clip"])
@pytest.mark.parametrize("device", [None, ""])
def test_missing_device_is_an_internal_error(cls, device):
    from marqo_b200 import loaders
    from marqo_b200.errors import InternalError
    with pytest.raises(InternalError, match="`device` is required for loading CLIP models!"):
        getattr(loaders, cls)(device=device, model_properties={"type": "clip"})


@pytest.mark.parametrize("source", [{"url": "https://example.com/m.pt"},
                                    {"model_location": {"s3": {"Bucket": "b", "Key": "k"}}}])
def test_download_sources_are_refused(source):
    from marqo_b200.errors import ModelLoadError
    from marqo_b200.loaders import B200Clip
    with pytest.raises(ModelLoadError, match="downloading the checkpoint is Marqo's job"):
        B200Clip(device="cuda:0", model_properties={"name": "m", "dimensions": 512, **source}).load()


@pytest.mark.parametrize("keys", [("localpath", "url"), ("localpath", "model_location"), ("url", "model_location")])
def test_more_than_one_source_is_refused(keys):
    from marqo_b200.errors import InvalidModelPropertiesError
    from marqo_b200.loaders import B200Clip
    props = {"name": "m", "dimensions": 512, **{k: "x" for k in keys}}
    with pytest.raises(InvalidModelPropertiesError, match="Only one of"):
        B200Clip(device="cuda:0", model_properties=props).load()


def test_missing_localpath_is_refused(tmp_path):
    from marqo_b200.errors import InvalidModelPropertiesError
    from marqo_b200.loaders import B200Clip
    with pytest.raises(InvalidModelPropertiesError, match="not a local file"):
        B200Clip(device="cuda:0", model_properties={"dimensions": 512, "localpath": str(tmp_path / "no.pt")}).load()


def test_preprocess_image_model():
    from marqo_b200 import model_registry as R, s2_inference as s2
    assert s2.is_preprocess_image_model(R.get_model_properties("ViT-B/32"))
    assert s2.is_preprocess_image_model(R.get_model_properties("RN101"))
    assert not s2.is_preprocess_image_model(R.get_model_properties("fp16/ViT-B/32"))
    assert s2.is_preprocess_image_model(s2.validate_model_properties("m", {"type": "clip", "dimensions": 512,
                                                                            "name": "ViT-B/16"}))
    assert not s2.is_preprocess_image_model(s2.validate_model_properties("m", {"type": "fp16_clip", "dimensions": 512,
                                                                                "name": "fp16/ViT-B/16"}))


def test_clip_tokenizer_is_the_bpe_at_77_from_merges_file():
    from marqo_b200.loaders import B200Clip
    import marqo_b200.tokenizers as T
    from marqo_b200 import model_registry as R
    for arch in (R.WIDE_RESNET_ARCHS["RN50x16"], R.get_model_properties("ViT-L/14@336px")["arch"]):
        m = B200Clip(device="cuda:0", model_properties={"merges_file": "unused"})
        m.arch = arch
        seen = {}

        class Tok:
            def __init__(self, path, context_length):
                seen["ctx"] = context_length

        orig = T.ClipBpeTokenizer
        T.ClipBpeTokenizer = Tok
        try:
            m._default_tokenizer()
        finally:
            T.ClipBpeTokenizer = orig
        assert seen["ctx"] == 77


def test_fp16_loader_rounds_to_float16(monkeypatch):
    from marqo_b200 import loaders
    vals = np.array([[1.0 + 2 ** -12, 0.3, -1e-3, 65504.0]], np.float32)
    monkeypatch.setattr(loaders.B200OpenCLIP, "encode_text", lambda self, s, normalize=True: vals)
    monkeypatch.setattr(loaders.B200OpenCLIP, "encode_image", lambda self, s, image_download_headers=None,
                        normalize=True: vals)
    m = loaders.B200Fp16Clip(device="cuda:0", model_properties={})
    for out in (m.encode("text"), m.encode_text("text"), m.encode_image([np.zeros((4, 4, 3), np.uint8)])):
        assert out.dtype == np.float16
        np.testing.assert_array_equal(out, vals.astype(np.float16))


# ------------------------------------------------------------------------------------------------------------------
# The arch from an OpenAI-format state dict's shapes
# ------------------------------------------------------------------------------------------------------------------
def _shape(*s):
    return np.broadcast_to(np.float32(0), s)   # shapes only: no memory


def _openai_shapes(arch):
    """{name: zero-memory array} with the names and shapes of OpenAI's CLIP state dicts (clip/model.py) for arch."""
    sd = {"logit_scale": _shape()}
    E = arch["embed_dim"]
    t = arch["text"] if "text" in arch else {k: arch[k] for k in ("width", "layers", "heads", "mlp", "ctx", "vocab")}

    def blocks(prefix, w, n):
        for i in range(n):
            p = f"{prefix}transformer.resblocks.{i}."
            sd.update({p + "attn.in_proj_weight": _shape(3 * w, w), p + "attn.in_proj_bias": _shape(3 * w),
                       p + "attn.out_proj.weight": _shape(w, w), p + "attn.out_proj.bias": _shape(w),
                       p + "ln_1.weight": _shape(w), p + "ln_1.bias": _shape(w), p + "ln_2.weight": _shape(w),
                       p + "ln_2.bias": _shape(w), p + "mlp.c_fc.weight": _shape(4 * w, w),
                       p + "mlp.c_fc.bias": _shape(4 * w), p + "mlp.c_proj.weight": _shape(w, 4 * w),
                       p + "mlp.c_proj.bias": _shape(w)})

    if "vision" in arch:
        v = arch["vision"]
        w, p, g = v["width"], v["patch"], v["image_size"] // v["patch"]
        sd.update({"visual.conv1.weight": _shape(w, 3, p, p), "visual.class_embedding": _shape(w),
                   "visual.positional_embedding": _shape(g * g + 1, w), "visual.ln_pre.weight": _shape(w),
                   "visual.ln_pre.bias": _shape(w), "visual.ln_post.weight": _shape(w),
                   "visual.ln_post.bias": _shape(w), "visual.proj": _shape(w, E)})
        blocks("visual.", w, v["layers"])
    else:
        r = arch["resnet"]
        w = r["width"]
        bn = lambda p, c: {f"{p}.{k}": _shape(c) for k in ("weight", "bias", "running_mean", "running_var")}
        for i, (cin, cout) in enumerate(((3, w // 2), (w // 2, w // 2), (w // 2, w)), start=1):
            sd[f"visual.conv{i}.weight"] = _shape(cout, cin, 3, 3)
            sd.update(bn(f"visual.bn{i}", cout))
        inplanes = w
        for s, depth in enumerate(r["layers"]):
            planes = w << s
            for i in range(depth):
                p = f"visual.layer{s + 1}.{i}."
                for j, (cin, cout, k) in enumerate(((inplanes, planes, 1), (planes, planes, 3),
                                                    (planes, 4 * planes, 1)), 1):
                    sd[f"{p}conv{j}.weight"] = _shape(cout, cin, k, k)
                    sd.update(bn(f"{p}bn{j}", cout))
                if i == 0:
                    sd[f"{p}downsample.0.weight"] = _shape(4 * planes, inplanes, 1, 1)
                    sd.update(bn(f"{p}downsample.1", 4 * planes))
                inplanes = 4 * planes
        C, g = 32 * w, r["image_size"] // 32
        sd["visual.attnpool.positional_embedding"] = _shape(g * g + 1, C)
        for nm, out_f in (("q_proj", C), ("k_proj", C), ("v_proj", C), ("c_proj", E)):
            sd[f"visual.attnpool.{nm}.weight"], sd[f"visual.attnpool.{nm}.bias"] = _shape(out_f, C), _shape(out_f)
    tw = t["width"]
    sd.update({"token_embedding.weight": _shape(t["vocab"], tw), "positional_embedding": _shape(t["ctx"], tw),
               "ln_final.weight": _shape(tw), "ln_final.bias": _shape(tw), "text_projection": _shape(tw, E)})
    blocks("", tw, t["layers"])
    return sd


def _arch(name):
    from marqo_b200 import model_registry as R
    return R.WIDE_RESNET_ARCHS[name] if name in WIDE else R.get_model_properties(name)["arch"]


@pytest.mark.parametrize("name", SERVED + list(WIDE))
def test_arch_from_openai_state_dict(name):
    from marqo_b200 import model_registry as R
    arch = _arch(name)
    assert R.openai_clip_arch(_openai_shapes(arch)) == arch


def test_rn50x4_stem_and_planes():
    """RN50x4's and RN50x16's stem channels, bottleneck planes and widest trunk output follow from their widths."""
    from marqo_b200 import model_registry as R
    a4, a16 = R.WIDE_RESNET_ARCHS["RN50x4"]["resnet"], R.WIDE_RESNET_ARCHS["RN50x16"]["resnet"]
    assert R.WIDE_RESNET_ARCHS["RN50x4"]["resnet"] == {"layers": [4, 6, 10, 6], "width": 80, "heads": 40,
                                                      "image_size": 288}
    for r, stem, planes, widest in ((a4, (40, 80), (80, 160, 320, 640), 2560),
                                    (a16, (48, 96), (96, 192, 384, 768), 3072)):
        w = r["width"]
        assert (w // 2, w) == stem and tuple(w << s for s in range(4)) == planes and 32 * w == widest
        assert r["heads"] * 64 == 32 * w


class _Holder(torch.nn.Module):
    """A scriptable module whose state dict is sd (dotted names become submodules)."""

    def __init__(self, sd):
        super().__init__()
        for name, v in sd.items():
            mod = self
            *path, leaf = name.split(".")
            for p in path:
                if not hasattr(mod, p):
                    mod.add_module(p, torch.nn.Module())
                mod = getattr(mod, p)
            mod.register_parameter(leaf, torch.nn.Parameter(torch.as_tensor(v), requires_grad=False))
        self.register_buffer("input_resolution", torch.tensor(224))   # OpenAI archives carry ints too

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return x


def test_torchscript_archive_loads_through_load_state_dict(tmp_path):
    from marqo_b200 import model_registry as R
    from marqo_b200.weights import load_state_dict, random_clip_weights
    arch = R._clip_arch(64, 64, 2, 1, 16, 64, 2, 1, act="quickgelu", image_size=32)
    arch["text"].update(ctx=8, vocab=50)
    sd = random_clip_weights(arch, seed=4)
    sd["logit_scale"] = np.float32(4.6).reshape(())
    # OpenAI's archives hold fp16 weights
    m = torch.jit.script(_Holder({k: torch.from_numpy(np.asarray(v)).half() for k, v in sd.items()}))
    path = tmp_path / "ViT-tiny.pt"
    torch.jit.save(m, str(path))
    got = load_state_dict(str(path))
    assert set(got) == set(sd)
    for k, v in sd.items():
        assert got[k].dtype == np.float32
        np.testing.assert_array_equal(got[k], np.asarray(v).astype(np.float16).astype(np.float32))
    assert R.openai_clip_arch(got) == arch
    # a plain torch.save state dict still goes through torch.load(weights_only=True)
    torch.save({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, str(tmp_path / "plain.pt"))
    assert set(load_state_dict(str(tmp_path / "plain.pt"))) == set(sd)


def test_custom_checkpoint_arch_reaches_the_encoder(monkeypatch, tmp_path):
    """A custom `clip` model with a localpath and no arch: B200Clip reads the checkpoint, infers the arch, and builds
    the encoder from both (the Encoder itself replaced by a recorder: no GPU here)."""
    from marqo_b200 import engine, loaders, model_registry as R
    from marqo_b200.weights import random_clip_resnet_weights
    arch = _arch("RN50x4")
    small = R._resnet_arch([1, 1, 1, 1], 640, "quickgelu", 80, 64, (64, 1, 1))
    small.update(ctx=8, vocab=50)
    sd = random_clip_resnet_weights(small, seed=2)
    path = tmp_path / "RN50x4-small.npz"
    np.savez(path, **sd)
    seen = {}

    class Rec:
        def __init__(self, kind, a, w, device=0, max_batch=256):
            seen.update(kind=kind, arch=a, keys=set(w), max_batch=max_batch)

    monkeypatch.setattr(engine, "Encoder", Rec)
    m = loaders.B200Clip(device="cuda:0", model_properties={"name": "mine", "dimensions": 640,
                                                             "localpath": str(path)})
    m.load()
    assert seen["kind"] == "clip_resnet" and seen["arch"] == small and seen["keys"] == set(sd)
    assert seen["max_batch"] == loaders.WIDE_RESNET_MAX_BATCH
    assert arch["resnet"]["width"] == small["resnet"]["width"]
    # the loader keeps the path and the inferred arch, not the state dict it read (Marqo caches loaders)
    assert m.model_properties["localpath"] == str(path) and m.model_properties["arch"] == small
    assert not any(isinstance(v, dict) and "text_projection" in v for v in m.model_properties.values())


def _small_clip_checkpoint(tmp_path, **change):
    from marqo_b200 import model_registry as R
    from marqo_b200.weights import random_clip_weights
    arch = R._clip_arch(64, 64, 1, 1, 16, 64, 1, 1, act="quickgelu", image_size=32)
    arch["text"].update(ctx=8, vocab=50)
    sd = {**random_clip_weights(arch, seed=5), **change}
    path = tmp_path / "clip.npz"
    np.savez(path, **{k: v for k, v in sd.items() if v is not None})
    return path


def test_declared_dimensions_must_match_the_checkpoint(tmp_path):
    from marqo_b200.errors import InvalidModelPropertiesError
    from marqo_b200.loaders import B200Clip
    path = _small_clip_checkpoint(tmp_path)
    m = B200Clip(device="cuda:0", model_properties={"name": "m", "dimensions": 512, "localpath": str(path)})
    with pytest.raises(InvalidModelPropertiesError, match="dimensions 512.*embeddings of 64"):
        m.load()


def test_non_openai_checkpoint_is_refused_by_name(tmp_path):
    """An open_clip checkpoint of another layout (here without ln_final, as the timm / HF text towers name it
    otherwise) is refused with the name it lacks, not a bare KeyError."""
    from marqo_b200.errors import InvalidModelPropertiesError
    from marqo_b200.loaders import B200Clip
    path = _small_clip_checkpoint(tmp_path, **{"ln_final.weight": None})
    m = B200Clip(device="cuda:0", model_properties={"name": "m", "dimensions": 64, "localpath": str(path)})
    with pytest.raises(InvalidModelPropertiesError, match="no `ln_final.weight`"):
        m.load()


# ------------------------------------------------------------------------------------------------------------------
# The fp32 oracle at the wide ResNets' widths
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("width", [80, 96])
def test_resnet_oracle_matches_torch_modules_at_width(width):
    from test_resnet_clip import _ResNet
    from marqo_b200 import model_registry as R
    from marqo_b200.weights import random_clip_resnet_weights
    layers, size = (1, 2, 1, 1), 64
    arch = R._resnet_arch(list(layers), 96, "quickgelu", width, size)
    arch["layers"] = 0
    sd = random_clip_resnet_weights(arch, seed=width)
    pixels = torch.randn(2, 3, size, size, generator=torch.Generator().manual_seed(width))
    got = O.encode_image(sd, arch, pixels, normalize=False)
    with torch.no_grad():
        ref = _ResNet(layers, width, width // 2, 96, size).load(sd, layers)(pixels)
    torch.testing.assert_close(got, ref, rtol=1e-5, atol=1e-5 * float(ref.abs().max()))
