"""EVA02 CLIP on the CPU: the registry entries against the reference's property dicts, the table lookups, the arch
blocks, the seeded weights' checkpoint names and shapes, the model size Marqo derives, the oracle's RoPE against an
independent complex-number formulation, the oracle's block against one built from nn.LayerNorm, F.silu and
F.scaled_dot_product_attention, and the preprocessing at 224 and 336 against torchvision's."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import _eva02_oracle as V
from oracle import encoders as E

# The reference's entries (src/marqo/s2_inference/model_registry.py:441-461); `type` is the engine's loader type.
REFERENCE = {
    V.B16: {"name": V.B16, "dimensions": 512, "note": "open_clip model: EVA02-B-16/merged2b_s8b_b131k",
            "type": "open_clip", "pretrained": "merged2b_s8b_b131k"},
    V.L14: {"name": V.L14, "dimensions": 768, "note": "open_clip model: EVA02-L-14/merged2b_s4b_b131k",
            "type": "open_clip", "pretrained": "merged2b_s4b_b131k"},
    V.L14_336: {"name": V.L14_336, "dimensions": 768, "note": "open_clip model: EVA02-L-14-336/merged2b_s6b_b61k",
                "type": "open_clip", "pretrained": "merged2b_s6b_b61k"},
}

# (trunk width, layers, heads, SwiGLU hidden, patch, image, text width, layers, heads, embed): the module docstring
ARCH = {
    V.B16: (768, 12, 12, 2048, 16, 224, 512, 12, 8, 512),
    V.L14: (1024, 24, 16, 2730, 14, 224, 768, 12, 12, 768),
    V.L14_336: (1024, 24, 16, 2730, 14, 336, 768, 12, 12, 768),
}


@pytest.mark.parametrize("name", V.NAMES)
def test_registry_entries(name):
    from marqo_b200 import model_registry as R
    p = R.get_model_properties(name)
    a = p.pop("arch")
    assert p == dict(REFERENCE[name], type=R.TYPE_OPEN_CLIP)
    w, layers, heads, hid, patch, image, tw, tl, th, embed = ARCH[name]
    assert hid == int(w * 4 * 2 / 3)
    assert a == {"kind": "clip_eva", "embed_dim": embed, "act": "gelu", "mean": R.OPENAI_MEAN, "std": R.OPENAI_STD,
                 "width": tw, "layers": tl, "heads": th, "mlp": 4 * tw, "ctx": 77, "vocab": 49408,
                 "eva": {"width": w, "layers": layers, "heads": heads, "mlp": hid, "patch": patch, "image_size": image,
                         "ln_eps": 1e-6, "rope_ref_grid": 16}}
    assert w // heads == 64


def test_tables():
    """EVA02_MODELS is reached by find_model and get_model_properties, and is in all_models() and served_models()."""
    from marqo_b200 import model_registry as R
    assert set(R.EVA02_MODELS) == set(V.NAMES)
    others = (R.MODELS, R.MPNET_MODELS, R.SIGLIP_MODELS, R.XLMR_MODELS, R.RESNET_MODELS, R.CONVNEXT_MODELS,
              R.BIG_VIT_MODELS)
    for name in V.NAMES:
        assert R.find_model(name) is R.EVA02_MODELS[name]
        assert not any(name in t for t in others)
        assert R.all_models()[name] is R.EVA02_MODELS[name]
        assert R.served_models()[name] is R.EVA02_MODELS[name]
        assert R.get_model_properties(name) == R.EVA02_MODELS[name]
        assert R.get_model_properties(name) is not R.EVA02_MODELS[name]
    assert set(R.served_models()) == set(R.all_models()) | set(R.CONVNEXT_MODELS) | set(R.BIG_VIT_MODELS)


def test_text_towers_are_served_gemm_shapes():
    """The top-level layout gives the GEMM shape tests only the text towers, whose (width, mlp) are served already."""
    from marqo_b200 import model_registry as R
    shapes = {(e["arch"]["width"], e["arch"]["mlp"]) for e in R.EVA02_MODELS.values()}
    assert shapes == {(512, 2048), (768, 3072)}
    assert all("vision" not in e["arch"] for e in R.EVA02_MODELS.values())


def test_model_size_comes_from_the_type():
    """No model_size in the entries, and no entry of Marqo's name table matches: 1 GB, the open_clip type's size."""
    from marqo_b200 import model_registry as R, s2_inference as s2
    for name in V.NAMES:
        assert "model_size" not in R.get_model_properties(name)
        assert s2.get_model_size(name, R.get_model_properties(name)) == 1


def test_loader_kind_and_random_weights():
    from marqo_b200 import loaders
    from marqo_b200.weights import random_eva02_weights
    a = V.arch(V.L14, eva_layers=1, text_layers=1)
    sd = loaders._resolve_weights({"random_init": 3}, a, "clip_eva")
    assert sd.keys() == random_eva02_weights(a, 3).keys()


def test_random_weights_have_the_checkpoint_names_and_shapes():
    a = V.arch(V.L14_336, eva_layers=2, text_layers=1)
    sd = V.weights(a, 1)
    W, H, E_, G = 1024, 2730, 768, 24
    t = "visual.trunk."
    want = {t + "patch_embed.proj.weight": (W, 3, 14, 14), t + "patch_embed.proj.bias": (W,),
            t + "cls_token": (1, 1, W), t + "pos_embed": (1, G * G + 1, W), t + "norm.weight": (W,),
            t + "norm.bias": (W,), t + "head.weight": (E_, W), t + "head.bias": (E_,)}
    for i in range(2):
        b = f"{t}blocks.{i}."
        want.update({b + "norm1.weight": (W,), b + "norm1.bias": (W,), b + "attn.q_proj.weight": (W, W),
                     b + "attn.q_proj.bias": (W,), b + "attn.k_proj.weight": (W, W), b + "attn.v_proj.weight": (W, W),
                     b + "attn.v_proj.bias": (W,), b + "attn.norm.weight": (W,), b + "attn.norm.bias": (W,),
                     b + "attn.proj.weight": (W, W), b + "attn.proj.bias": (W,), b + "norm2.weight": (W,),
                     b + "norm2.bias": (W,), b + "mlp.fc1_g.weight": (H, W), b + "mlp.fc1_g.bias": (H,),
                     b + "mlp.fc1_x.weight": (H, W), b + "mlp.fc1_x.bias": (H,), b + "mlp.norm.weight": (H,),
                     b + "mlp.norm.bias": (H,), b + "mlp.fc2.weight": (W, H), b + "mlp.fc2.bias": (W,)})
    got = {k: v.shape for k, v in sd.items() if k.startswith("visual.")}
    assert got == want
    assert "visual.trunk.blocks.0.attn.k_proj.bias" not in sd
    assert sd["text.text_projection"].shape == (768, 768)
    assert sd["text.token_embedding.weight"].shape == (49408, 768)
    assert sd["text.transformer.resblocks.0.attn.in_proj_weight"].shape == (3 * 768, 768)
    assert all(v.dtype == np.float32 for v in sd.values())


# ------------------------------------------------------------------------------------------------------------------
# RoPE
# ------------------------------------------------------------------------------------------------------------------
def _complex_rope(x, G, ref):
    """x [..., G*G, 64] rotated as complex numbers: pair i is x[2i] + i x[2i+1] times e^(i theta), theta of the
    module docstring, all in fp64."""
    r, c = torch.meshgrid(torch.arange(G, dtype=torch.float64), torch.arange(G, dtype=torch.float64), indexing="ij")
    s = ref / G
    j = torch.arange(32) % 16
    freq = 10000.0 ** (-j.double() / 16)
    p = torch.where(torch.arange(32) < 16, r.reshape(-1, 1) * s, c.reshape(-1, 1) * s)   # [G*G, 32]
    z = torch.view_as_complex(x.double().reshape(*x.shape[:-1], 32, 2).contiguous())
    out = z * torch.polar(torch.ones_like(p), p * freq)
    return torch.view_as_real(out).reshape(x.shape)


@pytest.mark.parametrize("G", [14, 16, 24])
def test_oracle_rope_matches_complex_rotation(G):
    x = torch.randn(3, G * G, 64, generator=torch.Generator().manual_seed(G))
    sin, cos = V.rope_sin_cos(G, 16)
    got = V.rotate(x, sin, cos)
    torch.testing.assert_close(got.double(), _complex_rope(x, G, 16), rtol=0, atol=2e-5)


@pytest.mark.parametrize("G,scale", [(14, 16 / 14), (16, 1.0), (24, 16 / 24)])
def test_rope_grid_scale_and_identity_at_the_origin(G, scale):
    """Grid position (0, 0) is the identity; pair 0 of position (1, 0) turns by s = 16 / G, pair 16 of (0, 1) too, and
    pair 1 of (1, 0) by s 10000^(-1/16)."""
    sin, cos = V.rope_sin_cos(G, 16)
    assert torch.equal(sin[0], torch.zeros(64)) and torch.equal(cos[0], torch.ones(64))
    theta = torch.atan2(sin, cos).double()
    assert math.isclose(theta[G, 0], scale, rel_tol=1e-6) and math.isclose(theta[G, 1], scale, rel_tol=1e-6)
    assert math.isclose(theta[1, 32], scale, rel_tol=1e-6) and math.isclose(theta[1, 33], scale, rel_tol=1e-6)
    assert theta[G, 32] == 0 and theta[1, 0] == 0   # rows turn the first 16 pairs, columns the last 16
    assert math.isclose(theta[G, 2], scale * 10000 ** (-1 / 16), rel_tol=1e-6)


def test_class_row_is_not_rotated():
    a = V.arch(V.B16, eva_layers=1, text_layers=0)
    sd = V.torch_sd(V.weights(a, 2), "visual.")
    x = torch.randn(2, 197, 768, generator=torch.Generator().manual_seed(1))
    sin, cos = V.rope_sin_cos(14, 16)
    p = "visual.trunk.blocks.0."
    # the class row's attention output depends on its q only through q itself: zeroing every patch row's rotation
    # (identity tables) must change the patch rows but leave the class row's q untouched
    got = V.block(x, sd, p, 12, sin, cos)
    ident = V.block(x, sd, p, 12, torch.zeros_like(sin), torch.ones_like(cos))
    assert not torch.allclose(got, ident)
    h = F.layer_norm(x, (768,), sd[p + "norm1.weight"], sd[p + "norm1.bias"], 1e-6)
    q = F.linear(h, sd[p + "attn.q_proj.weight"], sd[p + "attn.q_proj.bias"]).view(2, 197, 12, 64).transpose(1, 2)
    rq = torch.cat([q[:, :, :1], V.rotate(q[:, :, 1:], sin, cos)], dim=2)
    assert torch.equal(rq[:, :, 0], q[:, :, 0])


# ------------------------------------------------------------------------------------------------------------------
# The oracle's block against one built from torch modules
# ------------------------------------------------------------------------------------------------------------------
def _module_block(x, sd, p, heads, G, eps=1e-6):
    W = x.shape[-1]
    H = sd[p + "mlp.fc1_g.weight"].shape[0]

    def ln(name, n):
        m = torch.nn.LayerNorm(n, eps=eps)
        m.load_state_dict({"weight": sd[name + ".weight"], "bias": sd[name + ".bias"]})
        return m

    B, N, _ = x.shape
    h = ln(p + "norm1", W)(x)
    q = h @ sd[p + "attn.q_proj.weight"].t() + sd[p + "attn.q_proj.bias"]
    k = h @ sd[p + "attn.k_proj.weight"].t()
    v = h @ sd[p + "attn.v_proj.weight"].t() + sd[p + "attn.v_proj.bias"]
    q, k, v = (t.view(B, N, heads, 64).transpose(1, 2) for t in (q, k, v))
    q = torch.cat([q[:, :, :1], _complex_rope(q[:, :, 1:], G, 16).float()], dim=2)
    k = torch.cat([k[:, :, :1], _complex_rope(k[:, :, 1:], G, 16).float()], dim=2)
    o = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, N, W)
    x = x + ln(p + "attn.norm", W)(o) @ sd[p + "attn.proj.weight"].t() + sd[p + "attn.proj.bias"]
    h = ln(p + "norm2", W)(x)
    u = F.silu(h @ sd[p + "mlp.fc1_g.weight"].t() + sd[p + "mlp.fc1_g.bias"]) * (
        h @ sd[p + "mlp.fc1_x.weight"].t() + sd[p + "mlp.fc1_x.bias"])
    return x + ln(p + "mlp.norm", H)(u) @ sd[p + "mlp.fc2.weight"].t() + sd[p + "mlp.fc2.bias"]


@pytest.mark.parametrize("name,G", [(V.B16, 14), (V.L14, 16)])
@torch.no_grad()
def test_oracle_block_matches_torch_modules(name, G):
    a = V.arch(name, eva_layers=1, text_layers=0)
    ev = a["eva"]
    sd = V.torch_sd(V.weights(a, 4), "visual.")
    x = torch.randn(2, G * G + 1, ev["width"], generator=torch.Generator().manual_seed(G))
    sin, cos = V.rope_sin_cos(G, 16)
    got = V.block(x, sd, "visual.trunk.blocks.0.", ev["heads"], sin, cos)
    ref = _module_block(x, sd, "visual.trunk.blocks.0.", ev["heads"], G)
    torch.testing.assert_close(got, ref, rtol=1e-4, atol=1e-4)


# ------------------------------------------------------------------------------------------------------------------
# Preprocessing
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", [V.B16, V.L14_336])
@pytest.mark.parametrize("hw", [(480, 640), (640, 480), (100, 900)])
def test_preprocessing_crops_the_shortest_side(name, hw):
    """open_clip's image_transform for these models: torchvision Resize(S, BICUBIC) of the shortest side,
    CenterCrop(S), ToTensor, Normalize with the OpenAI statistics."""
    from PIL import Image
    from torchvision.transforms import CenterCrop, Compose, InterpolationMode, Normalize, Resize, ToTensor
    a = V.arch(name)
    S = a["eva"]["image_size"]
    h, w = hw
    img = np.random.default_rng(h + w).integers(0, 256, (2, h, w, 3), dtype=np.uint8)
    tf = Compose([Resize(S, interpolation=InterpolationMode.BICUBIC), CenterCrop(S), ToTensor(),
                  Normalize(E.OPENAI_CLIP_MEAN, E.OPENAI_CLIP_STD)])
    ref = torch.stack([tf(Image.fromarray(x)) for x in img])
    got = V.preprocess_u8(a, img)
    assert got.shape == (2, 3, S, S)
    torch.testing.assert_close(got, ref, rtol=0, atol=1e-6)
