"""fp32 torch restatement of LanguageBind's video model (LanguageBind/Video_V1.5_FT), written from the arithmetic the
reference runs, over a LanguageBindVideo state dict (transformers-style names, marqo_b200.weights.
random_languagebind_video_weights):

  video tower  languagebind/video/modeling_video.py:698-785 (CLIPVisionTransformer), layers :209-260
               (CLIPEncoderLayer with add_time_attn), embeddings :18-50 (vl) and :53-121 (vl_new, tube 1)
  text tower   modeling_video.py:555-640 (CLIPTextTransformer: causal mask, final_layer_norm, EOT = arg-max id)
  outputs      languagebind/__init__.py:55-64 (v / |v|, times exp(logit_scale) for non-language modalities) and
               multimodal_model_load.py:293-301 (Marqo's _normalize: / |v| again when normalize)
  transform    languagebind/video/processing_video.py:20-45, 80-93 (opencv backend): frame ids linspace(0, count - 1,
               T, dtype=int); x / 255; NormalizeVideo; pytorchvideo ShortSideScale (bilinear, align_corners False, no
               antialias; verify); CenterCropVideo (offsets int(round((size - S) / 2))); RandomHorizontalFlipVideo is
               left out (the engine does not flip).

Used by the CPU tests against the reference's own code (tests/golden/languagebind_golden.npz) and by the GPU tests
as the engine's yardstick.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

OPENAI_MEAN = (0.48145466, 0.4578275, 0.40821073)
OPENAI_STD = (0.26862954, 0.26130258, 0.27577711)
EPS = 1e-5


def _t(sd, k):
    v = sd[k]
    return v if isinstance(v, torch.Tensor) else torch.from_numpy(np.asarray(v, np.float32))


def _ln(x, sd, p):
    return F.layer_norm(x, (x.shape[-1],), _t(sd, p + "weight"), _t(sd, p + "bias"), EPS)


def _lin(x, sd, p, bias=True):
    y = x @ _t(sd, p + "weight").T
    return y + _t(sd, p + "bias") if bias else y


def _act(x, act):
    return x * torch.sigmoid(1.702 * x) if act == "quickgelu" else F.gelu(x)


def _mha(x, sd, p, heads, causal=False):
    """CLIPAttention: q, k, v, out projections with biases, scale head_dim^-0.5, optional causal mask."""
    B, L, W = x.shape
    hd = W // heads
    q, k, v = (_lin(x, sd, p + n + "_proj.").view(B, L, heads, hd).transpose(1, 2) for n in ("q", "k", "v"))
    s = (q * hd ** -0.5) @ k.transpose(-1, -2)
    if causal:
        s = s + torch.triu(torch.full((L, L), float("-inf"), device=x.device), 1)
    o = (torch.softmax(s, dim=-1) @ v).transpose(1, 2).reshape(B, L, W)
    return _lin(o, sd, p + "out_proj.")


def _block(x, sd, p, heads, act, causal=False):
    x = x + _mha(_ln(x, sd, p + "layer_norm1."), sd, p + "self_attn.", heads, causal)
    h = _lin(_act(_lin(_ln(x, sd, p + "layer_norm2."), sd, p + "mlp.fc1."), act), sd, p + "mlp.fc2.")
    return x + h


def video_pooled(sd, pixels, heads, act, layers):
    """pixels fp32 [B, T, 3, S, S] (transformed frames) -> the tower's pooled output [B, W]: ln_post of every frame's
    class row, then the mean over the frames."""
    vm = "vision_model."
    conv = _t(sd, vm + "embeddings.patch_embedding.weight")
    pixels = torch.as_tensor(pixels, dtype=torch.float32, device=conv.device)
    B, T = pixels.shape[:2]
    if conv.ndim == 5:   # Conv3d of tube 1
        conv = conv[:, :, 0]
    W, P = conv.shape[0], conv.shape[-1]
    x = F.conv2d(pixels.reshape(B * T, *pixels.shape[2:]), conv, stride=P).flatten(2).transpose(1, 2)
    cls = _t(sd, vm + "embeddings.class_embedding")
    cls = cls.expand(T, W) if cls.ndim == 1 else cls   # vl: one row for every frame; vl_new: row t for frame t
    x = torch.cat([cls.repeat(B, 1)[:, None, :], x], dim=1) + _t(sd, vm + "embeddings.position_embedding.weight")
    x = _ln(x, sd, vm + "pre_layrnorm.")
    N = x.shape[1]
    for i in range(layers):
        p = f"{vm}encoder.layers.{i}."
        if T != 1:   # the temporal embedding stays in the residual stream
            x = (x.view(B, T, N, W) + _t(sd, p + "temporal_embedding")[0, :T, None, :]).reshape(B * T, N, W)
        xt = x.view(B, T, N, W).permute(0, 2, 1, 3).reshape(B * N, T, W)
        o = _mha(_ln(xt, sd, p + "temporal_layer_norm1."), sd, p + "temporal_attn.", heads)
        x = x + o.view(B, N, T, W).permute(0, 2, 1, 3).reshape(B * T, N, W)
        x = _block(x, sd, p, heads, act)
    pooled = _ln(x[:, 0], sd, vm + "post_layernorm.")
    return pooled.view(B, T, W).mean(1)


def text_pooled(sd, ids, heads, act, layers):
    """ids int [n, S] -> final_layer_norm of each row's first arg-max token [n, W] (causal layers, no key mask)."""
    dev = _t(sd, "text_model.embeddings.token_embedding.weight").device
    ids = torch.as_tensor(np.asarray(ids), dtype=torch.long, device=dev)
    tm = "text_model."
    x = _t(sd, tm + "embeddings.token_embedding.weight")[ids]
    x = x + _t(sd, tm + "embeddings.position_embedding.weight")[: ids.shape[1]]
    for i in range(layers):
        x = _block(x, sd, f"{tm}encoder.layers.{i}.", heads, act, causal=True)
    x = _ln(x, sd, tm + "final_layer_norm.")
    return x[torch.arange(ids.shape[0], device=dev), ids.argmax(-1)]


def _unit(v):
    return v / v.norm(dim=-1, keepdim=True)


def encode_video(sd, pixels, heads, act, layers, normalize=True):
    v = _unit(video_pooled(sd, pixels, heads, act, layers) @ _t(sd, "visual_projection.weight").T)
    v = v * _t(sd, "logit_scale").reshape(()).exp()
    return (_unit(v) if normalize else v).cpu().numpy()


def encode_text(sd, ids, heads, act, layers, normalize=True):
    v = _unit(text_pooled(sd, ids, heads, act, layers) @ _t(sd, "text_projection.weight").T)
    return (_unit(v) if normalize else v).cpu().numpy()


# ---------------------------------------------------------------------------------------------------- transform
def resize_geometry(h, w, S):
    """(resized h, resized w, crop top, crop left): the short side to S, the long one floor(long / short * S); the
    centre crop's offsets int(round((size - S) / 2.0)) with Python's round (half to even)."""
    nh, nw = (int(math.floor(h / w * S)), S) if w < h else (S, int(math.floor(w / h * S)))
    return nh, nw, int(round((nh - S) / 2.0)), int(round((nw - S) / 2.0))


def _axis(n_in, n_out):
    """Bilinear taps of one axis, align_corners False: source scale (i + 0.5) - 0.5 with scale = n_in / n_out in
    fp32, the multiply-add rounded once (an fma: the fp64 product of two fp32 values and its difference with 0.5 are
    exact), clamped at 0; the far tap clamped to the last sample."""
    scale = np.float32(n_in) / np.float32(n_out)
    dst = np.arange(n_out, dtype=np.float32) + np.float32(0.5)
    src = np.maximum((dst.astype(np.float64) * np.float64(scale) - 0.5).astype(np.float32), np.float32(0))
    i0 = src.astype(np.int64)
    i1 = np.minimum(i0 + 1, n_in - 1)
    lam = (src - i0.astype(np.float32)).astype(np.float32)
    return torch.from_numpy(i0), torch.from_numpy(i1), torch.from_numpy(lam)


def transform(frames_u8, S=224, mean=OPENAI_MEAN, std=OPENAI_STD):
    """uint8 RGB frames [T, H, W, 3] -> fp32 [T, 3, S, S] in the reference's order: / 255, Normalize, the short-side
    bilinear resize, the centre crop."""
    x = torch.from_numpy(np.ascontiguousarray(frames_u8)).permute(0, 3, 1, 2).float() / 255.0
    x = (x - torch.tensor(mean).view(1, 3, 1, 1)) / torch.tensor(std).view(1, 3, 1, 1)
    T, _, h, w = x.shape
    nh, nw, top, left = resize_geometry(h, w, S)
    y0, y1, ly = _axis(h, nh)
    x0, x1, lx = _axis(w, nw)
    ly, lx = ly.view(-1, 1), lx.view(1, -1)
    rows0, rows1 = x[:, :, y0], x[:, :, y1]
    out = (1 - ly) * ((1 - lx) * rows0[..., x0] + lx * rows0[..., x1]) + ly * ((1 - lx) * rows1[..., x0] +
                                                                               lx * rows1[..., x1])
    return out[:, :, top:top + S, left:left + S].contiguous()


def frame_ids(count, T=8):
    """The frames the opencv backend reads: np.linspace(0, count - 1, T, dtype=int)."""
    return np.linspace(0, count - 1, T, dtype=int)
