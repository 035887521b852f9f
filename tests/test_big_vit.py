"""ViT-H-14, ViT-g-14 and ViT-bigG-14 CLIP on the CPU: the registry entries against the reference's property dicts, the
table lookups, the fp32 oracle at the three vision shapes against transformers' independent CLIP vision tower, and the
squash preprocessing of the DFN5B models against torchvision's."""
import numpy as np
import pytest
import torch

import _big_vit_oracle as B
from oracle import encoders as E

# The reference's entries (src/marqo/s2_inference/model_registry.py:237-256,378-384,392-398); `type` is the engine's
# loader type, as for every open_clip entry of the engine's registry.
REFERENCE = {
    B.H14: {"name": B.H14, "dimensions": 1024, "note": "open_clip models", "type": "open_clip",
            "pretrained": "laion2b_s32b_b79k"},
    B.G14: {"name": B.G14, "dimensions": 1024, "note": "open_clip models", "type": "open_clip",
            "pretrained": "laion2b_s12b_b42k"},
    B.G14_S34B: {"name": B.G14_S34B, "dimensions": 1024, "note": "open_clip models", "type": "open_clip",
                 "pretrained": "laion2b_s34b_b88k"},
    B.BIG_G: {"name": B.BIG_G, "dimensions": 1280, "note": "open_clip models", "type": "open_clip",
              "pretrained": "laion2b_s39b_b160k"},
    B.H14_378: {"name": B.H14_378, "dimensions": 1024, "note": "open_clip model: ViT-H-14-378-quickgelu/dfn5b",
                "type": "open_clip", "pretrained": "dfn5b"},
    B.H14_DFN: {"name": B.H14_DFN, "dimensions": 1024, "note": "open_clip model: ViT-H-14-quickgelu/dfn5b",
                "type": "open_clip", "pretrained": "dfn5b"},
}

# (vision width, layers, heads, mlp, image, act, resize, text width, layers, heads, embed) of the module docstring
ARCH = {
    B.H14: (1280, 32, 16, 5120, 224, "gelu", None, 1024, 24, 16, 1024),
    B.H14_DFN: (1280, 32, 16, 5120, 224, "quickgelu", "squash", 1024, 24, 16, 1024),
    B.H14_378: (1280, 32, 16, 5120, 378, "quickgelu", "squash", 1024, 24, 16, 1024),
    B.G14: (1408, 40, 16, 6144, 224, "gelu", None, 1024, 24, 16, 1024),
    B.G14_S34B: (1408, 40, 16, 6144, 224, "gelu", None, 1024, 24, 16, 1024),
    B.BIG_G: (1664, 48, 16, 8192, 224, "gelu", None, 1280, 32, 20, 1280),
}


@pytest.mark.parametrize("name", B.NAMES)
def test_registry_entries(name):
    from marqo_b200 import model_registry as R
    p = R.get_model_properties(name)
    a = p.pop("arch")
    assert p == dict(REFERENCE[name], type=R.TYPE_OPEN_CLIP)
    vw, vl, vh, vmlp, image, act, resize, tw, tl, th, embed = ARCH[name]
    assert a["vision"] == {"width": vw, "layers": vl, "heads": vh, "mlp": vmlp, "patch": 14, "image_size": image}
    assert a["text"] == {"width": tw, "layers": tl, "heads": th, "mlp": 4 * tw, "ctx": 77, "vocab": 49408}
    assert (a["embed_dim"], a["act"], a.get("resize_mode")) == (embed, act, resize)
    assert (a["mean"], a["std"]) == (R.OPENAI_MEAN, R.OPENAI_STD)
    assert "kind" not in a


def test_tables():
    """The names are in BIG_VIT_MODELS only: find_model, get_model_properties and served_models() reach them, and
    all_models() (the set the existing GEMM and attention shape tests enumerate) does not."""
    from marqo_b200 import model_registry as R
    assert set(R.BIG_VIT_MODELS) == set(B.NAMES)
    others = (R.MODELS, R.MPNET_MODELS, R.SIGLIP_MODELS, R.XLMR_MODELS, R.RESNET_MODELS, R.CONVNEXT_MODELS)
    for name in B.NAMES:
        assert R.find_model(name) is R.BIG_VIT_MODELS[name]
        assert not any(name in t for t in others)
        assert name not in R.all_models()
        assert R.served_models()[name] is R.BIG_VIT_MODELS[name]
    assert set(R.served_models()) == set(R.all_models()) | set(R.CONVNEXT_MODELS) | set(R.BIG_VIT_MODELS)


def test_model_size_comes_from_the_names():
    """No model_size in the entries: Marqo's name table gives 5 GB for vit-h / vit-g and 6 GB for vit-bigg-14."""
    from marqo_b200 import model_registry as R, s2_inference as s2
    sizes = {name: s2.get_model_size(name, R.get_model_properties(name)) for name in B.NAMES}
    assert sizes == {B.H14: 5, B.H14_DFN: 5, B.H14_378: 5, B.G14: 5, B.G14_S34B: 5, B.BIG_G: 6}


def test_other_open_clip_names_stay_unserved():
    from marqo_b200 import model_registry as R
    for name in ("open_clip/ViT-SO400M-14-SigLIP-384/webli",
                 "open_clip/xlm-roberta-large-ViT-H-14/frozen_laion5b_s13b_b90k", "open_clip/ViT-L-14-336/openai"):
        assert R.find_model(name) is None


def test_random_weights_have_the_checkpoint_shapes():
    from marqo_b200.weights import random_clip_weights
    a = B.arch(B.BIG_G, vision_layers=1, text_layers=1)
    sd = random_clip_weights(a)
    assert sd["visual.transformer.resblocks.0.attn.in_proj_weight"].shape == (3 * 1664, 1664)
    assert sd["visual.transformer.resblocks.0.attn.out_proj.weight"].shape == (1664, 1664)
    assert sd["visual.transformer.resblocks.0.mlp.c_fc.weight"].shape == (8192, 1664)
    assert sd["visual.positional_embedding"].shape == (257, 1664)
    assert sd["transformer.resblocks.0.attn.in_proj_weight"].shape == (3 * 1280, 1280)
    assert sd["visual.proj"].shape == (1664, 1280)


# ------------------------------------------------------------------------------------------------------------------
# The oracle against transformers.CLIPVisionModelWithProjection (2 layers of each vision shape)
# ------------------------------------------------------------------------------------------------------------------
def _hf_vision(cfg: E.ClipCfg, sd):
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection
    v = cfg.vision
    hc = CLIPVisionConfig(hidden_size=v.width, intermediate_size=v.mlp, num_hidden_layers=v.layers,
                          num_attention_heads=v.heads, image_size=v.image_size, patch_size=v.patch,
                          projection_dim=cfg.embed_dim, hidden_act="quick_gelu" if cfg.act == "quickgelu" else "gelu",
                          layer_norm_eps=1e-5, attention_dropout=0.0)
    model = CLIPVisionModelWithProjection(hc).eval()
    w = v.width
    m = {"vision_model.embeddings.class_embedding": sd["visual.class_embedding"],
         "vision_model.embeddings.patch_embedding.weight": sd["visual.conv1.weight"],
         "vision_model.embeddings.position_embedding.weight": sd["visual.positional_embedding"],
         "vision_model.pre_layrnorm.weight": sd["visual.ln_pre.weight"],
         "vision_model.pre_layrnorm.bias": sd["visual.ln_pre.bias"],
         "vision_model.post_layernorm.weight": sd["visual.ln_post.weight"],
         "vision_model.post_layernorm.bias": sd["visual.ln_post.bias"],
         "visual_projection.weight": sd["visual.proj"].t()}
    for i in range(v.layers):
        p, q = f"visual.transformer.resblocks.{i}.", f"vision_model.encoder.layers.{i}."
        for kind, src in (("weight", "attn.in_proj_weight"), ("bias", "attn.in_proj_bias")):
            for j, nm in enumerate(("q_proj", "k_proj", "v_proj")):
                m[q + f"self_attn.{nm}.{kind}"] = sd[p + src][j * w:(j + 1) * w]
        for kind in ("weight", "bias"):
            m[q + f"self_attn.out_proj.{kind}"] = sd[p + f"attn.out_proj.{kind}"]
            m[q + f"layer_norm1.{kind}"] = sd[p + f"ln_1.{kind}"]
            m[q + f"layer_norm2.{kind}"] = sd[p + f"ln_2.{kind}"]
            m[q + f"mlp.fc1.{kind}"] = sd[p + f"mlp.c_fc.{kind}"]
            m[q + f"mlp.fc2.{kind}"] = sd[p + f"mlp.c_proj.{kind}"]
    missing, unexpected = model.load_state_dict(m, strict=False)
    assert not unexpected and all("position_ids" in k for k in missing), (missing, unexpected)
    return model


@pytest.mark.parametrize("name", [B.H14, B.H14_378, B.G14, B.BIG_G])
def test_oracle_vision_matches_transformers(name):
    """Head dims 80, 88 and 104 at 257 and 730 tokens; QuickGELU at 378."""
    a = B.arch(name, vision_layers=2, text_layers=0)
    cfg = B.clip_cfg(a)
    sd = E.make_clip_weights(E.ClipCfg(cfg.embed_dim, cfg.vision, E.TowerCfg(64, 1, 1, 64, ctx=8, vocab=16),
                                       act=cfg.act), seed=len(name))
    S = cfg.vision.image_size
    pixels = torch.randn(2, 3, S, S, generator=torch.Generator().manual_seed(5))
    got = E.clip_encode_image(sd, cfg, pixels, normalize=False)
    with torch.no_grad():
        ref = _hf_vision(cfg, sd)(pixel_values=pixels).image_embeds
    torch.testing.assert_close(got, ref, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("hw", [(480, 640), (640, 480), (100, 900), (378, 378)])
def test_squash_preprocessing_at_378(hw):
    """The tests' squash preprocessing (PIL resize to 378 x 378, no crop) equals open_clip's resize_mode "squash"
    transform: torchvision Resize((378, 378), BICUBIC), ToTensor, Normalize with the OpenAI statistics."""
    from PIL import Image
    from torchvision.transforms import Compose, InterpolationMode, Normalize, Resize, ToTensor
    h, w = hw
    img = np.random.default_rng(h + w).integers(0, 256, (2, h, w, 3), dtype=np.uint8)
    tf = Compose([Resize((378, 378), interpolation=InterpolationMode.BICUBIC), ToTensor(),
                  Normalize(E.OPENAI_CLIP_MEAN, E.OPENAI_CLIP_STD)])
    ref = torch.stack([tf(Image.fromarray(a)) for a in img])
    got = B.preprocess_u8(B.arch(B.H14_378), img)
    assert got.shape == (2, 3, 378, 378)
    torch.testing.assert_close(got, ref, rtol=0, atol=1e-6)
    # the crop models keep the centre crop
    crop = B.preprocess_u8(B.arch(B.H14), img)
    torch.testing.assert_close(crop, E.clip_preprocess_u8(img, 224), rtol=0, atol=0)
