"""ORACLE — TEST INFRASTRUCTURE ONLY.  CPU fp32 restatement of the SigLIP forward the reference calls into, beside the
CLIP / BERT restatements of oracle/encoders.py.

The reference loads open_clip/ViT-{B,L}-16-SigLIP*/webli and Marqo/marqo-fashionSigLIP through open_clip 2.24.0 and
calls `encode_image` / `encode_text` (src/marqo/core/inference/embedding_models/open_clip_model.py:249-286) with its
SigLIP preprocessing branch (open_clip_model.py:92-93).  The arithmetic below restates open_clip's SigLIP model: a
timm `vit_*_siglip_*` trunk and open_clip's TextTransformer.  Neither package can be read offline, so the names and
shapes are (verify) items; the arithmetic is pinned to transformers' independent SigLIP implementation
(SiglipVisionModel / SiglipTextModel, tests/test_siglip.py):
  * vision: conv patch embedding with bias, + pos_embed (no class token, no ln_pre); pre-LN blocks (LayerNorm eps 1e-6,
    erf-GELU); final LayerNorm over every token; MAP head (timm AttentionPoolLatent, one latent): q = latent W_q^T +
    b_q, k|v = x W_kv^T + b_kv, softmax(q k^T / sqrt(hd)) v per head, proj, x + MLP(LN(x)); no projection
  * text: token + positional embedding, pre-LN blocks without a causal mask, ln_final, last position, Linear + bias
  * Marqo's fp32 cast + L2 normalise without an epsilon (abstract_clip_model.py:83-85)
  * preprocessing (open_clip pretrained._slpcfg): Resize((S, S), BICUBIC) on the PIL image (a squash, no crop),
    ToTensor, Normalize(0.5, 0.5)."""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict

import torch
import torch.nn.functional as F

SIGLIP_MEAN = (0.5, 0.5, 0.5)
SIGLIP_STD = (0.5, 0.5, 0.5)


@dataclass
class SiglipCfg:
    width: int = 768             # both towers, and the embedding (the vision tower has no projection)
    layers: int = 12
    heads: int = 12
    mlp: int = 3072              # blocks and the MAP head
    image_size: int = 224
    patch: int = 16
    ctx: int = 64
    vocab: int = 32000
    ln_eps: float = 1e-6

    @property
    def grid(self) -> int:
        return self.image_size // self.patch

    def arch(self) -> dict:
        """The registry's arch block of this shape (model_registry._siglip_arch)."""
        w = self.width
        return {"kind": "siglip", "embed_dim": w, "act": "gelu", "mean": SIGLIP_MEAN, "std": SIGLIP_STD,
                "resize_mode": "squash", "ln_eps": self.ln_eps,
                "vision": {"width": w, "layers": self.layers, "heads": self.heads, "mlp": self.mlp,
                           "patch": self.patch, "image_size": self.image_size, "map_mlp": self.mlp},
                "text": {"width": w, "layers": self.layers, "heads": self.heads, "mlp": self.mlp, "ctx": self.ctx,
                         "vocab": self.vocab}}


def tiny_siglip(image_size: int = 224) -> SiglipCfg:
    return SiglipCfg(width=128, layers=2, heads=2, mlp=512, image_size=image_size, vocab=1000)


# ------------------------------------------------------------------------------------------------ weights
def _lin(g, out_f, in_f, gain=1.0):
    return torch.randn(out_f, in_f, generator=g) * (gain / math.sqrt(in_f))


def _vec(g, n, std=0.1, mean=0.0):
    return mean + std * torch.randn(n, generator=g)


def _block(g, p: str, w: int, mlp: int, rg: float, names: tuple, sd: Dict[str, torch.Tensor]):
    ln1, qkv_w, qkv_b, out, ln2, fc, proj = names
    sd[p + ln1 + ".weight"] = _vec(g, w, 0.1, 1.0)
    sd[p + ln1 + ".bias"] = _vec(g, w)
    sd[p + qkv_w] = _lin(g, 3 * w, w, 1.5)
    sd[p + qkv_b] = _vec(g, 3 * w)
    sd[p + out + ".weight"] = _lin(g, w, w, rg)
    sd[p + out + ".bias"] = _vec(g, w)
    sd[p + ln2 + ".weight"] = _vec(g, w, 0.1, 1.0)
    sd[p + ln2 + ".bias"] = _vec(g, w)
    sd[p + fc + ".weight"] = _lin(g, mlp, w)
    sd[p + fc + ".bias"] = _vec(g, mlp)
    sd[p + proj + ".weight"] = _lin(g, w, mlp, rg)
    sd[p + proj + ".bias"] = _vec(g, w)


TIMM_NAMES = ("norm1", "attn.qkv.weight", "attn.qkv.bias", "attn.proj", "norm2", "mlp.fc1", "mlp.fc2")
OPEN_CLIP_NAMES = ("ln_1", "attn.in_proj_weight", "attn.in_proj_bias", "attn.out_proj", "ln_2", "mlp.c_fc",
                   "mlp.c_proj")


def make_siglip_weights(cfg: SiglipCfg, seed: int = 1234, text: bool = True) -> Dict[str, torch.Tensor]:
    """Seeded O(1)-activation random weights under open_clip's SigLIP state-dict names (text=False: the vision tower
    only)."""
    g = torch.Generator().manual_seed(seed)
    w, p, mlp = cfg.width, cfg.patch, cfg.mlp
    rg = 1.0 / math.sqrt(2.0 * cfg.layers)
    sd: Dict[str, torch.Tensor] = {}
    tr = "visual.trunk."
    sd[tr + "patch_embed.proj.weight"] = torch.randn(w, 3, p, p, generator=g) / math.sqrt(3 * p * p)
    sd[tr + "patch_embed.proj.bias"] = _vec(g, w)
    sd[tr + "pos_embed"] = 0.5 * torch.randn(1, cfg.grid * cfg.grid, w, generator=g)
    for i in range(cfg.layers):
        _block(g, f"{tr}blocks.{i}.", w, mlp, rg, TIMM_NAMES, sd)
    sd[tr + "norm.weight"] = _vec(g, w, 0.1, 1.0)
    sd[tr + "norm.bias"] = _vec(g, w)
    a = tr + "attn_pool."
    sd[a + "latent"] = torch.randn(1, 1, w, generator=g)
    sd[a + "q.weight"] = _lin(g, w, w, 1.5)
    sd[a + "q.bias"] = _vec(g, w)
    sd[a + "kv.weight"] = _lin(g, 2 * w, w, 1.5)
    sd[a + "kv.bias"] = _vec(g, 2 * w)
    sd[a + "proj.weight"] = _lin(g, w, w)
    sd[a + "proj.bias"] = _vec(g, w)
    sd[a + "norm.weight"] = _vec(g, w, 0.1, 1.0)
    sd[a + "norm.bias"] = _vec(g, w)
    sd[a + "mlp.fc1.weight"] = _lin(g, mlp, w)
    sd[a + "mlp.fc1.bias"] = _vec(g, mlp)
    sd[a + "mlp.fc2.weight"] = _lin(g, w, mlp)
    sd[a + "mlp.fc2.bias"] = _vec(g, w)
    if not text:
        return sd
    sd["text.token_embedding.weight"] = torch.randn(cfg.vocab, w, generator=g)
    sd["text.positional_embedding"] = 0.5 * torch.randn(cfg.ctx, w, generator=g)
    for i in range(cfg.layers):
        _block(g, f"text.transformer.resblocks.{i}.", w, mlp, rg, OPEN_CLIP_NAMES, sd)
    sd["text.ln_final.weight"] = _vec(g, w, 0.1, 1.0)
    sd["text.ln_final.bias"] = _vec(g, w)
    sd["text.text_projection.weight"] = _lin(g, w, w)
    sd["text.text_projection.bias"] = _vec(g, w)
    return sd


# ------------------------------------------------------------------------------------------------ forward
def _attend(q, k, v, heads: int) -> torch.Tensor:
    """q [B, Sq, W], k / v [B, S, W] -> softmax(q k^T / sqrt(hd)) v per head, [B, Sq, W]."""
    B, Sq, W = q.shape
    hd = W // heads
    q = q.view(B, Sq, heads, hd).transpose(1, 2)
    k = k.view(B, -1, heads, hd).transpose(1, 2)
    v = v.view(B, -1, heads, hd).transpose(1, 2)
    att = ((q / math.sqrt(hd)) @ k.transpose(-1, -2)).softmax(dim=-1)
    return (att @ v).transpose(1, 2).reshape(B, Sq, W)


def _blocks(x, sd, prefix: str, count: int, cfg: SiglipCfg, names: tuple) -> torch.Tensor:
    ln1, qkv_w, qkv_b, out, ln2, fc, proj = names
    w, eps = cfg.width, cfg.ln_eps
    for i in range(count):
        p = f"{prefix}{i}."
        h = F.layer_norm(x, (w,), sd[p + ln1 + ".weight"], sd[p + ln1 + ".bias"], eps)
        q, k, v = F.linear(h, sd[p + qkv_w], sd[p + qkv_b]).split(w, dim=-1)
        x = x + F.linear(_attend(q, k, v, cfg.heads), sd[p + out + ".weight"], sd[p + out + ".bias"])
        h = F.layer_norm(x, (w,), sd[p + ln2 + ".weight"], sd[p + ln2 + ".bias"], eps)
        h = F.gelu(F.linear(h, sd[p + fc + ".weight"], sd[p + fc + ".bias"]))
        x = x + F.linear(h, sd[p + proj + ".weight"], sd[p + proj + ".bias"])
    return x


def _l2_normalize(out: torch.Tensor) -> torch.Tensor:
    return out / out.norm(dim=-1, keepdim=True)      # abstract_clip_model.py:83-85: no epsilon


@torch.no_grad()
def siglip_encode_image(sd, cfg: SiglipCfg, pixels: torch.Tensor, normalize: bool = True) -> torch.Tensor:
    """pixels: fp32 [B, 3, S, S] already preprocessed -> [B, width]."""
    tr, w = "visual.trunk.", cfg.width
    x = F.conv2d(pixels.float(), sd[tr + "patch_embed.proj.weight"], sd[tr + "patch_embed.proj.bias"],
                 stride=cfg.patch)
    B = x.shape[0]
    x = x.reshape(B, w, -1).permute(0, 2, 1) + sd[tr + "pos_embed"]
    x = _blocks(x, sd, tr + "blocks.", cfg.layers, cfg, TIMM_NAMES)
    x = F.layer_norm(x, (w,), sd[tr + "norm.weight"], sd[tr + "norm.bias"], cfg.ln_eps)
    a = tr + "attn_pool."
    q = F.linear(sd[a + "latent"].reshape(1, 1, w), sd[a + "q.weight"], sd[a + "q.bias"]).expand(B, 1, w)
    k, v = F.linear(x, sd[a + "kv.weight"], sd[a + "kv.bias"]).split(w, dim=-1)
    o = F.linear(_attend(q, k, v, cfg.heads), sd[a + "proj.weight"], sd[a + "proj.bias"])
    h = F.layer_norm(o, (w,), sd[a + "norm.weight"], sd[a + "norm.bias"], cfg.ln_eps)
    o = o + F.linear(F.gelu(F.linear(h, sd[a + "mlp.fc1.weight"], sd[a + "mlp.fc1.bias"])), sd[a + "mlp.fc2.weight"],
                     sd[a + "mlp.fc2.bias"])
    out = o[:, 0].to(torch.float32)
    return _l2_normalize(out) if normalize else out


@torch.no_grad()
def siglip_encode_text(sd, cfg: SiglipCfg, ids: torch.Tensor, normalize: bool = True) -> torch.Tensor:
    """ids: int [B, seq] (open_clip pads to ctx = 64) -> [B, width]: no causal mask, the last position is pooled."""
    ids = ids.long()
    S = ids.shape[1]
    x = sd["text.token_embedding.weight"][ids] + sd["text.positional_embedding"][:S]
    x = _blocks(x, sd, "text.transformer.resblocks.", cfg.layers, cfg, OPEN_CLIP_NAMES)
    x = F.layer_norm(x, (cfg.width,), sd["text.ln_final.weight"], sd["text.ln_final.bias"], cfg.ln_eps)
    out = F.linear(x[:, -1], sd["text.text_projection.weight"], sd["text.text_projection.bias"]).to(torch.float32)
    return _l2_normalize(out) if normalize else out


# ------------------------------------------------------------------------------------------------ preprocess
def siglip_preprocess_pil(img, n_px: int) -> torch.Tensor:
    """open_clip's SigLIP image transform: Resize((n_px, n_px), BICUBIC) -> RGB -> ToTensor -> Normalize(0.5, 0.5)."""
    from torchvision.transforms import Compose, InterpolationMode, Normalize, Resize, ToTensor
    tf = Compose([Resize((n_px, n_px), interpolation=InterpolationMode.BICUBIC), lambda im: im.convert("RGB"),
                  ToTensor(), Normalize(SIGLIP_MEAN, SIGLIP_STD)])
    return tf(img)


def siglip_preprocess_u8(hwc_u8, n_px: int) -> torch.Tensor:
    """uint8 [n, H, W, 3] numpy -> fp32 [n, 3, n_px, n_px] through PIL."""
    from PIL import Image
    return torch.stack([siglip_preprocess_pil(Image.fromarray(a), n_px) for a in hwc_u8])
