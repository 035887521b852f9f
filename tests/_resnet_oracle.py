"""fp32 torch restatement of OpenAI's ResNet CLIP image tower (open_clip ModifiedResNet, verify) over its state dict:
functional conv, BatchNorm (eval), average pooling and F.multi_head_attention_forward.  The text tower is the CLIP text
transformer of oracle/encoders.py.  Preprocessing is the CLIP one (shortest side -> S bicubic, centre crop), as
oracle/encoders.clip_preprocess_u8 restates it."""
from __future__ import annotations

import torch
import torch.nn.functional as F

BN_EPS = 1e-5


def _bn(x, sd, p):
    return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"],
                        training=False, eps=BN_EPS)


def _conv_bn_relu(x, sd, conv, bn, stride=1, relu=True):
    w = sd[conv + ".weight"]
    y = _bn(F.conv2d(x, w, stride=stride, padding=w.shape[-1] // 2), sd, bn)
    return F.relu(y) if relu else y


def bottleneck(x, sd, p, stride):
    out = _conv_bn_relu(x, sd, p + "conv1", p + "bn1")
    out = _conv_bn_relu(out, sd, p + "conv2", p + "bn2")
    if stride > 1:
        out = F.avg_pool2d(out, stride)
    out = _conv_bn_relu(out, sd, p + "conv3", p + "bn3", relu=False)
    identity = x
    if p + "downsample.0.weight" in sd:
        identity = F.avg_pool2d(x, stride) if stride > 1 else x
        identity = _conv_bn_relu(identity, sd, p + "downsample.0", p + "downsample.1", relu=False)
    return F.relu(out + identity)


def trunk(sd, layers, pixels):
    """Stem and the four stages: fp32 NCHW [n, 3, S, S] (normalised) -> [n, 32 width, S/32, S/32]."""
    v = "visual."
    x = _conv_bn_relu(pixels, sd, v + "conv1", v + "bn1", stride=2)
    x = _conv_bn_relu(x, sd, v + "conv2", v + "bn2")
    x = _conv_bn_relu(x, sd, v + "conv3", v + "bn3")
    x = F.avg_pool2d(x, 2)
    for s, depth in enumerate(layers):
        for i in range(depth):
            x = bottleneck(x, sd, f"{v}layer{s + 1}.{i}.", 2 if (i == 0 and s > 0) else 1)
    return x


def attnpool(sd, x, heads):
    """AttentionPool2d: tokens [mean; pixels] + positional_embedding, multi-head attention with separate q/k/v
    projections, token 0 out."""
    a = "visual.attnpool."
    n, C, H, W = x.shape
    t = x.flatten(2).permute(2, 0, 1)                              # (HW, n, C)
    t = torch.cat([t.mean(dim=0, keepdim=True), t], dim=0)
    t = t + sd[a + "positional_embedding"][:, None, :]
    out, _ = F.multi_head_attention_forward(
        query=t[:1], key=t, value=t, embed_dim_to_check=C, num_heads=heads,
        q_proj_weight=sd[a + "q_proj.weight"], k_proj_weight=sd[a + "k_proj.weight"],
        v_proj_weight=sd[a + "v_proj.weight"], in_proj_weight=None,
        in_proj_bias=torch.cat([sd[a + "q_proj.bias"], sd[a + "k_proj.bias"], sd[a + "v_proj.bias"]]),
        bias_k=None, bias_v=None, add_zero_attn=False, dropout_p=0.0,
        out_proj_weight=sd[a + "c_proj.weight"], out_proj_bias=sd[a + "c_proj.bias"],
        use_separate_proj_weight=True, training=False, need_weights=False)
    return out[0]


def encode_image(sd, arch, pixels, normalize=True):
    """arch: the registry's clip_resnet block; pixels fp32 NCHW, already normalised."""
    sd = {k: torch.as_tensor(v).float().to(pixels.device) for k, v in sd.items() if k.startswith("visual.")}
    r = arch["resnet"]
    with torch.no_grad():
        y = attnpool(sd, trunk(sd, r["layers"], pixels.float()), r["heads"])
    return y / y.norm(dim=-1, keepdim=True) if normalize else y


def fold_bn(w, gamma, beta, mean, var, eps=BN_EPS):
    """BatchNorm folded into the conv before it, in fp64: (w', b') with conv(x, w') + b' == BN(conv(x, w))."""
    s = gamma.double() / torch.sqrt(var.double() + eps)
    return w.double() * s[:, None, None, None], beta.double() - mean.double() * s
