"""The ViT-H-14, ViT-g-14 and ViT-bigG-14 CLIP models for the tests: registry names, the oracle's config of an arch
block, reduced-depth archs and the squash preprocessing of the DFN5B models (oracle/encoders.py runs any head dim)."""
import numpy as np
import torch

from oracle import encoders as E

H14 = "open_clip/ViT-H-14/laion2b_s32b_b79k"
H14_DFN = "open_clip/ViT-H-14-quickgelu/dfn5b"
H14_378 = "open_clip/ViT-H-14-378-quickgelu/dfn5b"
G14 = "open_clip/ViT-g-14/laion2b_s12b_b42k"
G14_S34B = "open_clip/ViT-g-14/laion2b_s34b_b88k"
BIG_G = "open_clip/ViT-bigG-14/laion2b_s39b_b160k"
NAMES = (H14, H14_DFN, H14_378, G14, G14_S34B, BIG_G)
# one name per distinct (vision shape, activation, resize): the two ViT-g-14 tags share everything
SHAPES = (H14, H14_DFN, H14_378, G14, BIG_G)


def arch(name, vision_layers=None, text_layers=None):
    """A copy of the registry's arch block; layers None keeps the depth, 0 drops the tower."""
    from marqo_b200 import model_registry as R
    a = R.get_model_properties(name)["arch"]
    for tower, layers in (("vision", vision_layers), ("text", text_layers)):
        if layers == 0:
            a[tower] = None
        elif layers is not None:
            a[tower]["layers"] = layers
    return a


def clip_cfg(a) -> E.ClipCfg:
    """The oracle's ClipCfg of an arch block (a dropped tower becomes a 1-layer placeholder the oracle never runs)."""
    def tower(t, **kw):
        if t is None:
            return E.TowerCfg(64, 1, 1, 64, **kw)
        return E.TowerCfg(t["width"], t["layers"], t["heads"], t["mlp"], ctx=t.get("ctx", 0), vocab=t.get("vocab", 0),
                          image_size=t.get("image_size", 224), patch=t.get("patch", 0))
    return E.ClipCfg(a["embed_dim"], tower(a["vision"]), tower(a["text"]), act=a["act"], mean=tuple(a["mean"]),
                     std=tuple(a["std"]))


def squash_preprocess_u8(hwc_u8, S, mean=E.OPENAI_CLIP_MEAN, std=E.OPENAI_CLIP_STD) -> torch.Tensor:
    """uint8 [n, H, W, 3] -> fp32 [n, 3, S, S]: PIL resize((S, S), BICUBIC), ToTensor, Normalize (open_clip's
    resize_mode "squash")."""
    from PIL import Image
    out = []
    for a in hwc_u8:
        r = np.asarray(Image.fromarray(a).resize((S, S), Image.BICUBIC), dtype=np.float32) / 255.0
        t = torch.from_numpy(r).permute(2, 0, 1)
        out.append((t - torch.tensor(mean).view(3, 1, 1)) / torch.tensor(std).view(3, 1, 1))
    return torch.stack(out)


def preprocess_u8(a, hwc_u8) -> torch.Tensor:
    """The reference preprocessing of an arch: squash for resize_mode "squash", else shortest side + centre crop."""
    S = a["vision"]["image_size"]
    if a.get("resize_mode") == "squash":
        return squash_preprocess_u8(hwc_u8, S, a["mean"], a["std"])
    return E.clip_preprocess_u8(hwc_u8, S, a["mean"], a["std"])
