"""fp32 torch restatement of OWL-ViT's text-queried detection (transformers OwlViTForObjectDetection, verify), from a
state dict under the checkpoint's names, and of the reference's post-processing and per-image rerank loop.

The image is a float [3, S, S] tensor normalised by CLIP's mean and std, what OwlViTProcessor gives after its squash.
With G = S / patch:
  vision: conv (no bias) + class row, + positions, pre_layrnorm, pre-LN QuickGELU layers (eps 1e-5);
  e = post_layernorm(all rows); f_p = layer_norm(e_p * e_0) for p = 1 .. G^2 (row-major);
  text: token + position embeddings, causal QuickGELU layers, final_layer_norm of the row at argmax(id),
  text_projection (no bias), then / |.| (OwlViTModel's text_embeds);
  logit_p = (c^ . q^ + shift(f_p)) * (ELU(scale(f_p)) + 1), c^ = c / (|c| + 1e-6), q^ = t / (|t| + 1e-6);
  box_p = sigmoid(dense2(GELU(dense1(GELU(dense0(f_p))))) + box_bias[p]).
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

MEAN = (0.48145466, 0.4578275, 0.40821073)
STD = (0.26862954, 0.26130258, 0.27577711)


def _t(sd, k):
    v = sd[k]
    return (v if isinstance(v, torch.Tensor) else torch.from_numpy(v)).float()


def _layers(sd, prefix, x, heads, causal):
    L = len({k[len(prefix):].split(".")[0] for k in sd if k.startswith(prefix)})
    B, S, W = x.shape
    hd = W // heads
    mask = torch.full((S, S), float("-inf")).triu(1) if causal else None
    for i in range(L):
        p = f"{prefix}{i}."
        h = F.layer_norm(x, (W,), _t(sd, p + "layer_norm1.weight"), _t(sd, p + "layer_norm1.bias"), 1e-5)
        q, k, v = (F.linear(h, _t(sd, p + f"self_attn.{n}_proj.weight"), _t(sd, p + f"self_attn.{n}_proj.bias"))
                   .view(B, S, heads, hd).transpose(1, 2) for n in "qkv")
        a = (q * hd ** -0.5) @ k.transpose(-1, -2)
        if mask is not None:
            a = a + mask
        o = (a.softmax(-1) @ v).transpose(1, 2).reshape(B, S, W)
        x = x + F.linear(o, _t(sd, p + "self_attn.out_proj.weight"), _t(sd, p + "self_attn.out_proj.bias"))
        h = F.layer_norm(x, (W,), _t(sd, p + "layer_norm2.weight"), _t(sd, p + "layer_norm2.bias"), 1e-5)
        h = F.linear(h, _t(sd, p + "mlp.fc1.weight"), _t(sd, p + "mlp.fc1.bias"))
        h = h * torch.sigmoid(1.702 * h)
        x = x + F.linear(h, _t(sd, p + "mlp.fc2.weight"), _t(sd, p + "mlp.fc2.bias"))
    return x


def text_embed(sd, ids, heads):
    """The query's unit text embedding [n, E] from ids int [n, ctx]."""
    ids = torch.as_tensor(ids).long()
    tm = "owlvit.text_model."
    x = _t(sd, tm + "embeddings.token_embedding.weight")[ids] + \
        _t(sd, tm + "embeddings.position_embedding.weight")[: ids.shape[1]]
    x = _layers(sd, tm + "encoder.layers.", x, heads, causal=True)
    W = x.shape[-1]
    x = F.layer_norm(x, (W,), _t(sd, tm + "final_layer_norm.weight"), _t(sd, tm + "final_layer_norm.bias"), 1e-5)
    pooled = x[torch.arange(x.shape[0]), ids.to(torch.int).argmax(-1)]
    t = F.linear(pooled, _t(sd, "owlvit.text_projection.weight"))
    return t / torch.linalg.norm(t, dim=-1, keepdim=True)


def merged_features(sd, pixels, heads):
    """f [n, G^2, W] (the detector's patch features) of normalised images [n, 3, S, S]."""
    vm = "owlvit.vision_model."
    pre = "pre_layrnorm." if vm + "pre_layrnorm.weight" in sd else "pre_layernorm."
    cw = _t(sd, vm + "embeddings.patch_embedding.weight")
    p = cw.shape[-1]
    x = F.conv2d(pixels.float(), cw, stride=p).flatten(2).transpose(1, 2)
    W = x.shape[-1]
    cls = _t(sd, vm + "embeddings.class_embedding").expand(x.shape[0], 1, W)
    x = torch.cat([cls, x], 1) + _t(sd, vm + "embeddings.position_embedding.weight")
    x = F.layer_norm(x, (W,), _t(sd, vm + pre + "weight"), _t(sd, vm + pre + "bias"), 1e-5)
    x = _layers(sd, vm + "encoder.layers.", x, heads, causal=False)
    e = F.layer_norm(x, (W,), _t(sd, vm + "post_layernorm.weight"), _t(sd, vm + "post_layernorm.bias"), 1e-5)
    f = e[:, 1:] * e[:, :1]
    return F.layer_norm(f, (W,), _t(sd, "layer_norm.weight"), _t(sd, "layer_norm.bias"), 1e-5)


def box_bias(G: int) -> torch.Tensor:
    """compute_box_bias(G, G) in fp32, as transformers builds it."""
    xs = torch.arange(1, G + 1, dtype=torch.float32) / G
    xx, yy = torch.meshgrid(xs, xs, indexing="xy")
    c = torch.stack((xx, yy), -1).view(-1, 2).clip(0.0, 1.0)
    cb = torch.log(c + 1e-4) - torch.log1p(-c + 1e-4)
    s = torch.full_like(cb, 1.0 / G)
    sb = torch.log(s + 1e-4) - torch.log1p(-s + 1e-4)
    return torch.cat([cb, sb], -1)


def heads_from_features(sd, f, t):
    """(logits [n, G^2], boxes [n, G^2, 4]) from f [n, G^2, W] and the unit query t [E]."""
    c = F.linear(f, _t(sd, "class_head.dense0.weight"), _t(sd, "class_head.dense0.bias"))
    c = c / (torch.linalg.norm(c, dim=-1, keepdim=True) + 1e-6)
    q = t / (torch.linalg.norm(t, dim=-1, keepdim=True) + 1e-6)
    logit = c @ q
    shift = F.linear(f, _t(sd, "class_head.logit_shift.weight"), _t(sd, "class_head.logit_shift.bias"))[..., 0]
    scale = F.linear(f, _t(sd, "class_head.logit_scale.weight"), _t(sd, "class_head.logit_scale.bias"))[..., 0]
    logit = (logit + shift) * (F.elu(scale) + 1)
    h = F.gelu(F.linear(f, _t(sd, "box_head.dense0.weight"), _t(sd, "box_head.dense0.bias")))
    h = F.gelu(F.linear(h, _t(sd, "box_head.dense1.weight"), _t(sd, "box_head.dense1.bias")))
    b = F.linear(h, _t(sd, "box_head.dense2.weight"), _t(sd, "box_head.dense2.bias"))
    G = int(round(math.sqrt(f.shape[1])))
    return logit, torch.sigmoid(b + box_bias(G))


@torch.no_grad()
def detect(sd, pixels, ids, vision_heads, text_heads):
    """(logits [n, G^2], boxes [n, G^2, 4]) of normalised images [n, 3, S, S] against one query's ids [ctx]."""
    t = text_embed(sd, torch.as_tensor(ids).view(1, -1), text_heads)[0]
    return heads_from_features(sd, merged_features(sd, pixels, vision_heads), t)


def pixels_from_u8(hwc) -> torch.Tensor:
    """uint8 [n, S, S, 3] (already at the model's size) -> normalised fp32 [n, 3, S, S]."""
    x = torch.as_tensor(hwc).permute(0, 3, 1, 2).float() / 255.0
    return (x - torch.tensor(MEAN).view(1, 3, 1, 1)) / torch.tensor(STD).view(1, 3, 1, 1)


def post_process(logits, boxes, h: int, w: int):
    """transformers 4.41 OwlViTImageProcessor.post_process for one image and one query: (scores [P], corner boxes
    [P, 4] scaled to w x h)."""
    scores = torch.sigmoid(torch.as_tensor(logits))
    cx, cy, bw, bh = torch.as_tensor(boxes).unbind(-1)
    corners = torch.stack([cx - 0.5 * bw, cy - 0.5 * bh, cx + 0.5 * bw, cy + 0.5 * bh], dim=-1)
    return scores, corners * torch.tensor([w, h, w, h], dtype=torch.float32)[None, :]
