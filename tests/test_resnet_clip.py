"""OpenAI ResNet CLIP on the CPU: the registry entries against the reference's, the fp32 oracle (tests/_resnet_oracle.py)
against the same network built from torch modules, BatchNorm folding, the weight names the engine loads, and the
routing of vectorise("open_clip/RN50/openai") to the engine's open_clip loader."""
import numpy as np
import pytest
import torch
from torch import nn

import _resnet_oracle as O

# model_registry.py:80-126 of the reference: name -> (dimensions, pretrained)
REFERENCE = {
    "open_clip/RN50/openai": (1024, "openai"), "open_clip/RN50/yfcc15m": (1024, "yfcc15m"),
    "open_clip/RN50/cc12m": (1024, "cc12m"), "open_clip/RN50-quickgelu/openai": (1024, "openai"),
    "open_clip/RN50-quickgelu/yfcc15m": (1024, "yfcc15m"), "open_clip/RN50-quickgelu/cc12m": (1024, "cc12m"),
    "open_clip/RN101/openai": (512, "openai"), "open_clip/RN101/yfcc15m": (512, "yfcc15m"),
    "open_clip/RN101-quickgelu/openai": (512, "openai"), "open_clip/RN101-quickgelu/yfcc15m": (512, "yfcc15m"),
}


@pytest.mark.parametrize("name", sorted(REFERENCE))
def test_registry_entries(name):
    from marqo_b200 import model_registry as R
    e = R.get_model_properties(name)
    assert R.find_model(name) is R.RESNET_MODELS[name] and R.all_models()[name] is R.RESNET_MODELS[name]
    dims, tag = REFERENCE[name]
    assert (e["name"], e["dimensions"], e["pretrained"], e["type"]) == (name, dims, tag, R.TYPE_OPEN_CLIP)
    a = e["arch"]
    assert a["act"] == ("quickgelu" if tag == "openai" or "-quickgelu" in name else "gelu")
    assert "vision" not in a and a["kind"] == "clip_resnet" and a["embed_dim"] == dims
    assert (a["width"], a["layers"], a["heads"], a["mlp"], a["ctx"], a["vocab"]) == (512, 12, 8, 2048, 77, 49408)
    assert a["resnet"] == {"layers": [3, 4, 6, 3] if "RN50" in name else [3, 4, 23, 3], "width": 64, "heads": 32,
                           "image_size": 224}
    assert tuple(a["mean"]) == R.OPENAI_MEAN and tuple(a["std"]) == R.OPENAI_STD


def test_only_the_reference_resnets_are_served():
    from marqo_b200 import model_registry as R
    assert set(R.RESNET_MODELS) == set(REFERENCE)
    assert R.find_model("open_clip/RN50x4/openai") is None


# ------------------------------------------------------------------------------------------------------------------
# The oracle against torch modules
# ------------------------------------------------------------------------------------------------------------------
def _tiny_arch(layers=(1, 2, 1, 1), image_size=64, embed=96):
    from marqo_b200 import model_registry as R
    a = R._resnet_arch(list(layers), embed, "quickgelu")
    a["resnet"]["image_size"] = image_size
    a["layers"] = 0   # no text tower
    return a


class _Bottleneck(nn.Module):
    def __init__(self, inplanes, planes, stride):
        super().__init__()
        self.conv1, self.bn1 = nn.Conv2d(inplanes, planes, 1, bias=False), nn.BatchNorm2d(planes)
        self.conv2, self.bn2 = nn.Conv2d(planes, planes, 3, padding=1, bias=False), nn.BatchNorm2d(planes)
        self.avgpool = nn.AvgPool2d(stride) if stride > 1 else nn.Identity()
        self.conv3, self.bn3 = nn.Conv2d(planes, 4 * planes, 1, bias=False), nn.BatchNorm2d(4 * planes)
        self.downsample = None
        if stride > 1 or inplanes != 4 * planes:
            self.downsample = nn.Sequential(nn.AvgPool2d(stride), nn.Conv2d(inplanes, 4 * planes, 1, bias=False),
                                            nn.BatchNorm2d(4 * planes))
            # open_clip names the conv and the BN downsample.0 / .1 (its pool is parameter-free)

    def forward(self, x):
        out = torch.relu(self.bn1(self.conv1(x)))
        out = torch.relu(self.bn2(self.conv2(out)))
        out = self.bn3(self.conv3(self.avgpool(out)))
        identity = x if self.downsample is None else self.downsample(x)
        return torch.relu(out + identity)


class _ResNet(nn.Module):
    def __init__(self, layers, width, heads, embed, image_size):
        super().__init__()
        self.conv1, self.bn1 = nn.Conv2d(3, width // 2, 3, stride=2, padding=1, bias=False), nn.BatchNorm2d(width // 2)
        self.conv2, self.bn2 = nn.Conv2d(width // 2, width // 2, 3, padding=1, bias=False), nn.BatchNorm2d(width // 2)
        self.conv3, self.bn3 = nn.Conv2d(width // 2, width, 3, padding=1, bias=False), nn.BatchNorm2d(width)
        blocks, inplanes = [], width
        for s, depth in enumerate(layers):
            stage = []
            for i in range(depth):
                stage.append(_Bottleneck(inplanes, width << s, 2 if (i == 0 and s > 0) else 1))
                inplanes = 4 * (width << s)
            blocks.append(nn.Sequential(*stage))
        self.layers = nn.ModuleList(blocks)
        C, g = 32 * width, image_size // 32
        self.pos = nn.Parameter(torch.zeros(g * g + 1, C))
        self.mha = nn.MultiheadAttention(C, heads)
        self.c_proj = nn.Linear(C, embed)

    def forward(self, x):
        x = torch.relu(self.bn1(self.conv1(x)))
        x = torch.relu(self.bn2(self.conv2(x)))
        x = nn.functional.avg_pool2d(torch.relu(self.bn3(self.conv3(x))), 2)
        for stage in self.layers:
            x = stage(x)
        t = x.flatten(2).permute(2, 0, 1)
        t = torch.cat([t.mean(0, keepdim=True), t]) + self.pos[:, None, :]
        out, _ = self.mha(t[:1], t, t, need_weights=False)
        return self.c_proj(out[0])   # nn.MultiheadAttention's own out_proj is set to the identity below

    def load(self, sd, layers):
        v, a = "visual.", "visual.attnpool."
        t = {k: torch.from_numpy(x) for k, x in sd.items()}

        def bn(mod, p):
            mod.weight.data, mod.bias.data = t[p + ".weight"], t[p + ".bias"]
            mod.running_mean.data, mod.running_var.data = t[p + ".running_mean"], t[p + ".running_var"]

        for i in (1, 2, 3):
            getattr(self, f"conv{i}").weight.data = t[f"{v}conv{i}.weight"]
            bn(getattr(self, f"bn{i}"), f"{v}bn{i}")
        for s, stage in enumerate(self.layers):
            for i, blk in enumerate(stage):
                p = f"{v}layer{s + 1}.{i}."
                for j in (1, 2, 3):
                    getattr(blk, f"conv{j}").weight.data = t[f"{p}conv{j}.weight"]
                    bn(getattr(blk, f"bn{j}"), f"{p}bn{j}")
                if blk.downsample is not None:
                    blk.downsample[1].weight.data = t[p + "downsample.0.weight"]
                    bn(blk.downsample[2], p + "downsample.1")
        self.pos.data = t[a + "positional_embedding"]
        # the pool's separate q / k / v projections, stacked as the module's packed in-projection
        self.mha.in_proj_weight.data = torch.cat([t[a + "q_proj.weight"], t[a + "k_proj.weight"], t[a + "v_proj.weight"]])
        self.mha.in_proj_bias.data = torch.cat([t[a + "q_proj.bias"], t[a + "k_proj.bias"], t[a + "v_proj.bias"]])
        C = self.pos.shape[1]
        self.mha.out_proj.weight.data, self.mha.out_proj.bias.data = torch.eye(C), torch.zeros(C)
        self.c_proj.weight.data, self.c_proj.bias.data = t[a + "c_proj.weight"], t[a + "c_proj.bias"]
        return self.eval()


@pytest.mark.parametrize("layers,size", [((1, 2, 1, 1), 64), ((3, 4, 6, 3), 224)], ids=["tiny", "rn50"])
def test_oracle_matches_torch_modules(layers, size):
    from marqo_b200.weights import random_clip_resnet_weights
    arch = _tiny_arch(layers, size, 1024)
    sd = random_clip_resnet_weights(arch, seed=size)
    pixels = torch.randn(2, 3, size, size, generator=torch.Generator().manual_seed(1))
    got = O.encode_image(sd, arch, pixels, normalize=False)
    with torch.no_grad():
        ref = _ResNet(layers, 64, 32, 1024, size).load(sd, layers)(pixels)
    torch.testing.assert_close(got, ref, rtol=1e-5, atol=1e-5 * float(ref.abs().max()))


def test_bn_folding_in_fp64_equals_conv_then_bn():
    g = torch.Generator().manual_seed(3)
    w = torch.randn(32, 16, 3, 3, generator=g)
    gamma, beta, mean = torch.randn(32, generator=g), torch.randn(32, generator=g), torch.randn(32, generator=g)
    var = torch.rand(32, generator=g) + 0.1
    x = torch.randn(2, 16, 9, 9, generator=g).double()
    wf, bf = O.fold_bn(w, gamma, beta, mean, var)
    folded = torch.nn.functional.conv2d(x, wf, bf, padding=1)
    ref = torch.nn.functional.batch_norm(torch.nn.functional.conv2d(x, w.double(), padding=1), mean.double(),
                                         var.double(), gamma.double(), beta.double(), training=False, eps=O.BN_EPS)
    torch.testing.assert_close(folded, ref, rtol=1e-12, atol=1e-12)


def _required_names(layers, E):
    """The parameter names finalize reads (include/marqo_b200.h, CLIP ResNet) with their shapes."""
    bn = lambda p, c: {f"{p}.{k}": (c,) for k in ("weight", "bias", "running_mean", "running_var")}
    v, names = "visual.", {}
    for i, (cin, cout) in enumerate(((3, 32), (32, 32), (32, 64)), start=1):
        names[f"{v}conv{i}.weight"] = (cout, cin, 3, 3)
        names.update(bn(f"{v}bn{i}", cout))
    inplanes = 64
    for s, depth in enumerate(layers):
        planes = 64 << s
        for i in range(depth):
            p = f"{v}layer{s + 1}.{i}."
            for j, (cin, cout, k) in enumerate(((inplanes, planes, 1), (planes, planes, 3), (planes, 4 * planes, 1)), 1):
                names[f"{p}conv{j}.weight"] = (cout, cin, k, k)
                names.update(bn(f"{p}bn{j}", cout))
            if i == 0:
                names[f"{p}downsample.0.weight"] = (4 * planes, inplanes, 1, 1)
                names.update(bn(f"{p}downsample.1", 4 * planes))
            inplanes = 4 * planes
    a = v + "attnpool."
    names[a + "positional_embedding"] = (50, 2048)
    for nm, out_f in (("q_proj", 2048), ("k_proj", 2048), ("v_proj", 2048), ("c_proj", E)):
        names[f"{a}{nm}.weight"], names[f"{a}{nm}.bias"] = (out_f, 2048), (out_f,)
    return names


@pytest.mark.parametrize("name", ["open_clip/RN50/openai", "open_clip/RN101/yfcc15m"])
def test_random_weights_carry_the_names_finalize_requires(name):
    from marqo_b200 import model_registry as R
    from marqo_b200.weights import random_clip_resnet_weights, random_clip_weights
    arch = R.get_model_properties(name)["arch"]
    sd = random_clip_resnet_weights(arch, seed=1)
    visual = {k: tuple(v.shape) for k, v in sd.items() if k.startswith("visual.")}
    assert visual == _required_names(arch["resnet"]["layers"], arch["embed_dim"])
    clip_text = random_clip_weights({"embed_dim": arch["embed_dim"],
                                     "text": {k: arch[k] for k in ("width", "layers", "heads", "mlp", "ctx", "vocab")}})
    assert {k: tuple(v.shape) for k, v in sd.items() if not k.startswith("visual.")} == \
        {k: tuple(v.shape) for k, v in clip_text.items()}


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


@pytest.mark.parametrize("name,dims", [("open_clip/RN50/openai", 1024), ("open_clip/RN101-quickgelu/yfcc15m", 512)])
def test_vectorise_routes_resnets_to_the_open_clip_loader(monkeypatch, name, dims):
    from marqo_b200 import loaders, model_registry as R, s2_inference
    assert loaders.LOADERS[R.TYPE_OPEN_CLIP] is loaders.B200OpenCLIP
    monkeypatch.setitem(loaders.LOADERS, R.TYPE_OPEN_CLIP, _FakeLoader)
    monkeypatch.setattr(s2_inference, "_available_models", {})
    _FakeLoader.seen.clear()
    out = s2_inference.vectorise(name, "a photo of a dog", device="cuda:0")
    assert len(out) == 1 and len(out[0]) == dims
    (props,) = _FakeLoader.seen
    assert props["type"] == R.TYPE_OPEN_CLIP and props["arch"]["kind"] == "clip_resnet"


def test_clip_tokenizer_takes_ctx_from_the_top_level(tmp_path):
    from marqo_b200 import model_registry as R
    from marqo_b200.loaders import B200OpenCLIP
    m = B200OpenCLIP(device="cuda:0", model_properties={"merges_file": "unused"})
    m.arch = R.get_model_properties("open_clip/RN50/openai")["arch"]
    import marqo_b200.tokenizers as T
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
