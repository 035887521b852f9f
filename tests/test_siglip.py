"""SigLIP on the CPU: the fp32 oracle (tests/_siglip_oracle.py) against transformers' independent SigLIP towers, its
squash preprocessing against Pillow, the registry entries, the weight names the engine loads, and the routing of
vectorise("Marqo/marqo-fashionSigLIP") to the engine's open_clip loader."""
import numpy as np
import pytest
import torch

import _siglip_oracle as O

SIZES = [224, 64]


def _hf_vision(cfg: O.SiglipCfg, sd):
    from transformers import SiglipVisionConfig, SiglipVisionModel
    hc = SiglipVisionConfig(hidden_size=cfg.width, intermediate_size=cfg.mlp, num_hidden_layers=cfg.layers,
                            num_attention_heads=cfg.heads, image_size=cfg.image_size, patch_size=cfg.patch,
                            hidden_act="gelu", layer_norm_eps=cfg.ln_eps, attention_dropout=0.0)
    model = SiglipVisionModel(hc).eval()
    tr, a, w = "visual.trunk.", "visual.trunk.attn_pool.", cfg.width
    m = {"embeddings.patch_embedding.weight": sd[tr + "patch_embed.proj.weight"],
         "embeddings.patch_embedding.bias": sd[tr + "patch_embed.proj.bias"],
         "embeddings.position_embedding.weight": sd[tr + "pos_embed"][0],
         "post_layernorm.weight": sd[tr + "norm.weight"], "post_layernorm.bias": sd[tr + "norm.bias"],
         "head.probe": sd[a + "latent"],
         "head.attention.in_proj_weight": torch.cat([sd[a + "q.weight"], sd[a + "kv.weight"]]),
         "head.attention.in_proj_bias": torch.cat([sd[a + "q.bias"], sd[a + "kv.bias"]]),
         "head.attention.out_proj.weight": sd[a + "proj.weight"], "head.attention.out_proj.bias": sd[a + "proj.bias"],
         "head.layernorm.weight": sd[a + "norm.weight"], "head.layernorm.bias": sd[a + "norm.bias"]}
    for nm in ("fc1", "fc2"):
        for kind in ("weight", "bias"):
            m[f"head.mlp.{nm}.{kind}"] = sd[f"{a}mlp.{nm}.{kind}"]
    for i in range(cfg.layers):
        p, q = f"{tr}blocks.{i}.", f"encoder.layers.{i}."
        for kind in ("weight", "bias"):
            qkv = sd[p + f"attn.qkv.{kind}"]
            for j, nm in enumerate(("q_proj", "k_proj", "v_proj")):
                m[q + f"self_attn.{nm}.{kind}"] = qkv[j * w:(j + 1) * w]
            m[q + f"self_attn.out_proj.{kind}"] = sd[p + f"attn.proj.{kind}"]
            m[q + f"layer_norm1.{kind}"] = sd[p + f"norm1.{kind}"]
            m[q + f"layer_norm2.{kind}"] = sd[p + f"norm2.{kind}"]
            m[q + f"mlp.fc1.{kind}"] = sd[p + f"mlp.fc1.{kind}"]
            m[q + f"mlp.fc2.{kind}"] = sd[p + f"mlp.fc2.{kind}"]
    missing, unexpected = model.vision_model.load_state_dict(m, strict=False)
    assert not unexpected and all("position_ids" in k for k in missing), (missing, unexpected)
    return model


def _hf_text(cfg: O.SiglipCfg, sd):
    from transformers import SiglipTextConfig, SiglipTextModel
    hc = SiglipTextConfig(vocab_size=cfg.vocab, hidden_size=cfg.width, intermediate_size=cfg.mlp,
                          num_hidden_layers=cfg.layers, num_attention_heads=cfg.heads, max_position_embeddings=cfg.ctx,
                          hidden_act="gelu", layer_norm_eps=cfg.ln_eps, projection_size=cfg.width,
                          attention_dropout=0.0)
    model = SiglipTextModel(hc).eval()
    w = cfg.width
    m = {"embeddings.token_embedding.weight": sd["text.token_embedding.weight"],
         "embeddings.position_embedding.weight": sd["text.positional_embedding"],
         "final_layer_norm.weight": sd["text.ln_final.weight"], "final_layer_norm.bias": sd["text.ln_final.bias"],
         "head.weight": sd["text.text_projection.weight"], "head.bias": sd["text.text_projection.bias"]}
    for i in range(cfg.layers):
        p, q = f"text.transformer.resblocks.{i}.", f"encoder.layers.{i}."
        for kind, src in (("weight", "attn.in_proj_weight"), ("bias", "attn.in_proj_bias")):
            for j, nm in enumerate(("q_proj", "k_proj", "v_proj")):
                m[q + f"self_attn.{nm}.{kind}"] = sd[p + src][j * w:(j + 1) * w]
        for kind in ("weight", "bias"):
            m[q + f"self_attn.out_proj.{kind}"] = sd[p + f"attn.out_proj.{kind}"]
            m[q + f"layer_norm1.{kind}"] = sd[p + f"ln_1.{kind}"]
            m[q + f"layer_norm2.{kind}"] = sd[p + f"ln_2.{kind}"]
            m[q + f"mlp.fc1.{kind}"] = sd[p + f"mlp.c_fc.{kind}"]
            m[q + f"mlp.fc2.{kind}"] = sd[p + f"mlp.c_proj.{kind}"]
    missing, unexpected = model.text_model.load_state_dict(m, strict=False)
    assert not unexpected and all("position_ids" in k for k in missing), (missing, unexpected)
    return model


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("normalize", [True, False])
def test_oracle_vision_matches_transformers(size, normalize):
    cfg = O.tiny_siglip(size)
    sd = O.make_siglip_weights(cfg, seed=size)
    pixels = torch.randn(3, 3, size, size, generator=torch.Generator().manual_seed(7))
    got = O.siglip_encode_image(sd, cfg, pixels, normalize=normalize)
    with torch.no_grad():
        ref = _hf_vision(cfg, sd)(pixel_values=pixels).pooler_output
    if normalize:
        ref = ref / ref.norm(dim=-1, keepdim=True)
    torch.testing.assert_close(got, ref, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("seq", [64, 16])
@pytest.mark.parametrize("normalize", [True, False])
def test_oracle_text_matches_transformers(seq, normalize):
    cfg = O.tiny_siglip()
    sd = O.make_siglip_weights(cfg, seed=seq)
    ids = torch.randint(0, cfg.vocab, (3, seq), generator=torch.Generator().manual_seed(3))
    got = O.siglip_encode_text(sd, cfg, ids, normalize=normalize)
    with torch.no_grad():
        ref = _hf_text(cfg, sd)(input_ids=ids).pooler_output
    if normalize:
        ref = ref / ref.norm(dim=-1, keepdim=True)
    torch.testing.assert_close(got, ref, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("hw,S", [((37, 53), 224), ((301, 517), 224), ((101, 700), 256), ((500, 90), 384),
                                  ((224, 224), 224)],
                         ids=["upscale", "downscale", "x-down-y-up", "x-up-y-down", "identity"])
def test_preprocess_squashes_like_pillow(hw, S):
    from PIL import Image
    h, w = hw
    img = np.random.default_rng(h * w).integers(0, 256, (2, h, w, 3), dtype=np.uint8)
    got = O.siglip_preprocess_u8(img, S)
    ref = []
    for a in img:
        r = np.asarray(Image.fromarray(a).resize((S, S), Image.BICUBIC), dtype=np.float32) / 255.0
        ref.append(torch.from_numpy((r - 0.5) / 0.5).permute(2, 0, 1))
    assert got.shape == (2, 3, S, S)
    torch.testing.assert_close(got, torch.stack(ref), rtol=0, atol=1e-6)


# ------------------------------------------------------------------------------------------------------------------
# Registry, weights and routing
# ------------------------------------------------------------------------------------------------------------------
B16 = {"open_clip/ViT-B-16-SigLIP/webli": 224, "open_clip/ViT-B-16-SigLIP-256/webli": 256,
       "open_clip/ViT-B-16-SigLIP-384/webli": 384, "open_clip/ViT-B-16-SigLIP-512/webli": 512,
       "Marqo/marqo-fashionSigLIP": 224}
L16 = {"open_clip/ViT-L-16-SigLIP-256/webli": 256, "open_clip/ViT-L-16-SigLIP-384/webli": 384}


@pytest.mark.parametrize("name", sorted({**B16, **L16}))
def test_registry_entries(name):
    from marqo_b200 import model_registry as R
    e = R.get_model_properties(name)
    assert e == R.all_models()[name] and name in R.SIGLIP_MODELS
    w, layers, heads, size = (768, 12, 12, B16[name]) if name in B16 else (1024, 24, 16, L16[name])
    assert e["type"] == R.TYPE_OPEN_CLIP and e["dimensions"] == w
    a = e["arch"]
    assert (a["kind"], a["act"], a["resize_mode"], a["ln_eps"], a["embed_dim"]) == ("siglip", "gelu", "squash", 1e-6, w)
    assert tuple(a["mean"]) == tuple(a["std"]) == (0.5, 0.5, 0.5)
    assert a["vision"] == {"width": w, "layers": layers, "heads": heads, "mlp": 4 * w, "patch": 16, "image_size": size,
                           "map_mlp": 4 * w}
    assert a["text"] == {"width": w, "layers": layers, "heads": heads, "mlp": 4 * w, "ctx": 64, "vocab": 32000}
    if name == "Marqo/marqo-fashionSigLIP":
        assert e["name"] == "hf-hub:Marqo/marqo-fashionSigLIP" and "pretrained" not in e
    else:
        assert e["name"] == name and e["pretrained"] == "webli"


def test_so400m_is_not_served():
    from marqo_b200 import model_registry as R
    from marqo_b200.errors import UnknownModelError
    assert R.find_model("open_clip/ViT-SO400M-14-SigLIP-384/webli") is None
    with pytest.raises(UnknownModelError):
        R.get_model_properties("open_clip/ViT-SO400M-14-SigLIP-384/webli")


def test_random_weights_use_the_oracle_names_and_shapes():
    from marqo_b200.weights import random_siglip_weights
    cfg = O.tiny_siglip(64)
    ours = random_siglip_weights(cfg.arch(), seed=1)
    ref = O.make_siglip_weights(cfg)
    assert {k: tuple(v.shape) for k, v in ours.items()} == {k: tuple(v.shape) for k, v in ref.items()}


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


def test_vectorise_routes_fashion_siglip_to_the_open_clip_loader(monkeypatch):
    from marqo_b200 import loaders, model_registry as R, s2_inference
    assert loaders.LOADERS[R.TYPE_OPEN_CLIP] is loaders.B200OpenCLIP
    monkeypatch.setitem(loaders.LOADERS, R.TYPE_OPEN_CLIP, _FakeLoader)
    monkeypatch.setattr(s2_inference, "_available_models", {})
    _FakeLoader.seen.clear()
    out = s2_inference.vectorise("Marqo/marqo-fashionSigLIP", "a red dress", device="cuda:0")
    assert len(out) == 1 and len(out[0]) == 768
    (props,) = _FakeLoader.seen
    assert props["type"] == R.TYPE_OPEN_CLIP and props["arch"]["kind"] == "siglip"


def test_text_without_tokenizer_is_a_clear_error():
    from marqo_b200.errors import ModelLoadError
    from marqo_b200.loaders import B200OpenCLIP
    m = B200OpenCLIP(device="cuda:0", model_properties={})
    m.arch = O.tiny_siglip().arch()
    with pytest.raises(ModelLoadError, match="tokenizer"):
        m._tokenize("a red dress")
