"""The EVA02 CLIP models for the tests: registry names, reduced-depth archs and the fp32 torch restatement of the EVA02
image tower (open_clip TimmModel over timm's Eva; model_registry's docstring, verify).  The text tower is the CLIP one
of oracle/encoders.py under the "text." prefix."""
import math

import torch
import torch.nn.functional as F

from oracle import encoders as E

B16 = "open_clip/EVA02-B-16/merged2b_s8b_b131k"
L14 = "open_clip/EVA02-L-14/merged2b_s4b_b131k"
L14_336 = "open_clip/EVA02-L-14-336/merged2b_s6b_b61k"
NAMES = (B16, L14, L14_336)


def arch(name, eva_layers=None, text_layers=None):
    """A copy of the registry's arch block; layers None keeps the depth, 0 drops the tower."""
    from marqo_b200 import model_registry as R
    a = R.get_model_properties(name)["arch"]
    if eva_layers == 0:
        a["eva"] = None
    elif eva_layers is not None:
        a["eva"]["layers"] = eva_layers
    if text_layers is not None:
        a["layers"] = text_layers
    return a


def weights(a, seed):
    """Seeded weights of an arch block under the checkpoint names (marqo_b200.weights.random_eva02_weights)."""
    from marqo_b200.weights import random_eva02_weights
    return random_eva02_weights(a, seed=seed)


def torch_sd(sd, prefix, device="cpu"):
    return {k: torch.as_tensor(v).to(device) for k, v in sd.items() if k.startswith(prefix)}


# ------------------------------------------------------------------------------------------------ RoPE
def rope_sin_cos(G, ref=16, dtype=torch.float32):
    """timm build_rotary_pos_embed(feat_shape (G, G), dim 64, in_pixels False, ref_feat_shape (ref, ref)) -> (sin,
    cos), each [G * G, 64]: freq_bands 10000^(-j/16), the "ij" grid of positions scaled by ref / G, and
    repeat_interleave(2) so that columns 2i and 2i + 1 share pair i's angle."""
    bands = 1.0 / (10000 ** (torch.arange(0, 16, dtype=dtype) / 16))
    t = torch.arange(G, dtype=dtype) / G * ref
    grid = torch.stack(torch.meshgrid(t, t, indexing="ij"), dim=-1)     # [G, G, 2]: (row, column) positions
    pos = grid.unsqueeze(-1) * bands                                    # [G, G, 2, 16]
    sin = pos.sin().reshape(G * G, -1).repeat_interleave(2, -1)
    cos = pos.cos().reshape(G * G, -1).repeat_interleave(2, -1)
    return sin, cos


def rotate(x, sin, cos):
    """timm apply_rot_embed_cat: x cos + rot(x) sin, rot(x)[2i] = -x[2i+1], rot(x)[2i+1] = x[2i]."""
    rot = torch.stack([-x[..., 1::2], x[..., ::2]], -1).reshape(x.shape)
    return x * cos + rot * sin


# ------------------------------------------------------------------------------------------------ the tower
def block(x, sd, p, heads, sin, cos, eps=1e-6):
    """One timm EvaBlock (scale_attn_inner, SwiGLU with scale_mlp, no layer scale) over x [B, N, W], fp32."""
    B, N, W = x.shape
    hd = W // heads
    h = F.layer_norm(x, (W,), sd[p + "norm1.weight"], sd[p + "norm1.bias"], eps)
    q = F.linear(h, sd[p + "attn.q_proj.weight"], sd[p + "attn.q_proj.bias"])
    k = F.linear(h, sd[p + "attn.k_proj.weight"])
    v = F.linear(h, sd[p + "attn.v_proj.weight"], sd[p + "attn.v_proj.bias"])
    q, k, v = (t.view(B, N, heads, hd).transpose(1, 2) for t in (q, k, v))
    q = torch.cat([q[:, :, :1], rotate(q[:, :, 1:], sin, cos)], dim=2)
    k = torch.cat([k[:, :, :1], rotate(k[:, :, 1:], sin, cos)], dim=2)
    att = ((q / math.sqrt(hd)) @ k.transpose(-1, -2)).softmax(dim=-1)
    o = (att @ v).transpose(1, 2).reshape(B, N, W)
    o = F.layer_norm(o, (W,), sd[p + "attn.norm.weight"], sd[p + "attn.norm.bias"], eps)
    x = x + F.linear(o, sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"])
    h = F.layer_norm(x, (W,), sd[p + "norm2.weight"], sd[p + "norm2.bias"], eps)
    u = F.silu(F.linear(h, sd[p + "mlp.fc1_g.weight"], sd[p + "mlp.fc1_g.bias"])) * F.linear(
        h, sd[p + "mlp.fc1_x.weight"], sd[p + "mlp.fc1_x.bias"])
    u = F.layer_norm(u, (u.shape[-1],), sd[p + "mlp.norm.weight"], sd[p + "mlp.norm.bias"], eps)
    return x + F.linear(u, sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"])


@torch.no_grad()
def encode_image(sd, a, pixels, normalize=True):
    """pixels: fp32 [B, 3, S, S] already preprocessed -> the EVA02 image embeddings, Marqo's L2 rule when normalize."""
    ev = a["eva"]
    t = "visual.trunk."
    W, P = ev["width"], ev["patch"]
    G = ev["image_size"] // P
    dev = pixels.device
    x = F.conv2d(pixels.float(), sd[t + "patch_embed.proj.weight"], sd[t + "patch_embed.proj.bias"], stride=P)
    B = x.shape[0]
    x = x.reshape(B, W, -1).permute(0, 2, 1)
    x = torch.cat([sd[t + "cls_token"].expand(B, 1, W), x], dim=1) + sd[t + "pos_embed"]
    sin, cos = (r.to(dev) for r in rope_sin_cos(G, ev["rope_ref_grid"]))
    for i in range(ev["layers"]):
        x = block(x, sd, f"{t}blocks.{i}.", ev["heads"], sin, cos, ev["ln_eps"])
    x = F.layer_norm(x, (W,), sd[t + "norm.weight"], sd[t + "norm.bias"], ev["ln_eps"])
    out = F.linear(x[:, 0], sd[t + "head.weight"], sd[t + "head.bias"])
    return out / out.norm(dim=-1, keepdim=True) if normalize else out


def text_cfg(a) -> E.ClipCfg:
    """The oracle's ClipCfg of an arch's text tower (the vision tower a placeholder the text oracle never runs)."""
    text = E.TowerCfg(a["width"], a["layers"], a["heads"], a["mlp"], ctx=a["ctx"], vocab=a["vocab"])
    return E.ClipCfg(a["embed_dim"], E.TowerCfg(64, 1, 1, 64), text, act=a["act"])


@torch.no_grad()
def encode_text(sd, a, ids, normalize=True):
    """The CLIP text tower under the "text." prefix (text.text_projection is the [W, E] projection)."""
    tsd = {k[len("text."):]: torch.as_tensor(v) for k, v in sd.items() if k.startswith("text.")}
    return E.clip_encode_text(tsd, text_cfg(a), ids, normalize=normalize)


def preprocess_u8(a, hwc_u8) -> torch.Tensor:
    """open_clip's image_transform for these models: shortest side -> S (bicubic), centre crop, OpenAI mean / std."""
    return E.clip_preprocess_u8(hwc_u8, a["eva"]["image_size"], a["mean"], a["std"])
