"""fp32 torch restatement of the ConvNeXt CLIP image tower over its open_clip state dict (verify): timm's ConvNeXt trunk
(stem conv + LayerNorm, per stage a LayerNorm + 2 x 2 stride-2 downsample conv, blocks
x + gamma * fc2(GELU(fc1(LN(dwconv7x7(x))))), then global average pool + head.norm), open_clip TimmModel's head (a
Linear without bias, or an MLP: fc1 with bias, GELU, fc2 without bias) and Marqo's L2 normalisation.  Written from the
published architecture; tests/test_convnext_clip.py pins the trunk against transformers.ConvNextModel.  The text tower is
the CLIP text transformer of oracle/encoders.py, and preprocessing is the CLIP one (shortest side -> S bicubic, centre
crop), as oracle/encoders.clip_preprocess_u8 restates it."""
from __future__ import annotations

import torch
import torch.nn.functional as F


def _ln_channels(x, sd, p, eps):
    """LayerNorm over the channels of every pixel of NCHW x (timm LayerNorm2d)."""
    return F.layer_norm(x.permute(0, 2, 3, 1), (x.shape[1],), sd[p + ".weight"], sd[p + ".bias"], eps).permute(0, 3, 1, 2)


def block(x, sd, p, eps):
    C = x.shape[1]
    y = F.conv2d(x, sd[p + "conv_dw.weight"], sd[p + "conv_dw.bias"], padding=3, groups=C).permute(0, 2, 3, 1)
    y = F.layer_norm(y, (C,), sd[p + "norm.weight"], sd[p + "norm.bias"], eps)
    y = F.gelu(F.linear(y, sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"]))
    y = F.linear(y, sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"]) * sd[p + "gamma"]
    return x + y.permute(0, 3, 1, 2)


def trunk(sd, cx, pixels):
    """fp32 NCHW [n, 3, S, S] (normalised) -> [n, dims[3], S/32, S/32]; cx: the registry's "convnext" block."""
    t, eps = "visual.trunk.", cx["ln_eps"]
    x = F.conv2d(pixels, sd[t + "stem.0.weight"], sd[t + "stem.0.bias"], stride=4)
    x = _ln_channels(x, sd, t + "stem.1", eps)
    for s, depth in enumerate(cx["depths"]):
        p = f"{t}stages.{s}."
        if s > 0:
            x = _ln_channels(x, sd, p + "downsample.0", eps)
            x = F.conv2d(x, sd[p + "downsample.1.weight"], sd[p + "downsample.1.bias"], stride=2)
        for i in range(depth):
            x = block(x, sd, f"{p}blocks.{i}.", eps)
    return x


def pooled(sd, cx, pixels):
    """The trunk's output: LayerNorm (head.norm) of the mean over H x W."""
    x = trunk(sd, cx, pixels).mean(dim=(2, 3))
    t = "visual.trunk.head.norm"
    return F.layer_norm(x, (x.shape[1],), sd[t + ".weight"], sd[t + ".bias"], cx["ln_eps"])


def encode_image(sd, arch, pixels, normalize=True):
    """arch: the registry's clip_convnext block; pixels fp32 NCHW, already normalised."""
    sd = {k: torch.as_tensor(v).float().to(pixels.device) for k, v in sd.items() if k.startswith("visual.")}
    cx = arch["convnext"]
    with torch.no_grad():
        y = pooled(sd, cx, pixels.float())
        if cx["head"] == "mlp":
            h = F.gelu(F.linear(y, sd["visual.head.mlp.fc1.weight"], sd["visual.head.mlp.fc1.bias"]))
            y = F.linear(h, sd["visual.head.mlp.fc2.weight"])
        else:
            y = F.linear(y, sd["visual.head.proj.weight"])
    return y / y.norm(dim=-1, keepdim=True) if normalize else y


def to_hf(sd):
    """The trunk's open_clip names -> transformers.ConvNextModel's (the head norm becomes its final layernorm)."""
    out = {}
    for k, v in sd.items():
        if not k.startswith("visual.trunk."):
            continue
        k = k[len("visual.trunk."):]
        k = (k.replace("stem.0.", "embeddings.patch_embeddings.").replace("stem.1.", "embeddings.layernorm.")
             .replace("head.norm.", "layernorm.").replace("downsample.", "downsampling_layer.")
             .replace("blocks.", "layers.").replace("conv_dw.", "dwconv.").replace(".norm.", ".layernorm.")
             .replace("mlp.fc1.", "pwconv1.").replace("mlp.fc2.", "pwconv2.").replace(".gamma", ".layer_scale_parameter"))
        if k.startswith("stages."):
            k = "encoder." + k
        out[k] = torch.as_tensor(v)
    return out
