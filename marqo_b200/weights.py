"""Checkpoint plumbing for the encoders: state-dict loading and random initialisation.

The engine consumes parameters under their checkpoint names (open_clip state_dict names for CLIP, HF BertModel names
for BERT), so a real checkpoint loads unchanged: open_clip `*.pt/*.bin` state dicts, HF `pytorch_model.bin`, or an
`.npz` with the same keys.  `random_*` build seeded random-init weights of a given architecture (bench.py and the
service's self-test use them — there is no network for real checkpoints in the build environment)."""
from __future__ import annotations

import math
from typing import Dict

import numpy as np


def load_state_dict(path: str) -> Dict[str, np.ndarray]:
    """.npz, torch .pt/.bin/.pth or .safetensors -> {name: fp32 ndarray}."""
    p = str(path)
    if p.endswith(".npz"):
        with np.load(p) as z:
            return {k: np.asarray(z[k], dtype=np.float32) for k in z.files}
    if p.endswith(".safetensors"):
        from safetensors.numpy import load_file  # optional dependency
        return {k: np.asarray(v, dtype=np.float32) for k, v in load_file(p).items()}
    import torch
    sd = torch.load(p, map_location="cpu", weights_only=True)
    if isinstance(sd, dict) and "state_dict" in sd and isinstance(sd["state_dict"], dict):
        sd = sd["state_dict"]
    out = {}
    for k, v in sd.items():
        if hasattr(v, "is_floating_point") and v.is_floating_point():
            out[k[len("module."):] if k.startswith("module.") else k] = v.float().numpy()
    return out


def strip_hf_prefix(sd: Dict[str, np.ndarray]) -> Dict[str, np.ndarray]:
    """HF checkpoints saved from BertForXxx / MPNetForXxx / XLMRobertaForXxx carry a 'bert.' / 'mpnet.' / 'roberta.'
    prefix; BertModel, MPNetModel and XLMRobertaModel checkpoints do not."""
    for prefix in ("bert.", "mpnet.", "roberta."):
        if any(k.startswith(prefix) for k in sd):
            return {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}
    return sd


def _rng(seed):
    return np.random.default_rng(seed)


def _lin(g, out_f, in_f, gain=1.0):
    return (g.standard_normal((out_f, in_f), dtype=np.float32) * np.float32(gain / math.sqrt(in_f)))


def _vec(g, n, std=0.1, mean=0.0):
    return (mean + std * g.standard_normal(n, dtype=np.float32)).astype(np.float32)


def _clip_blocks(g, prefix, t, sd):
    w, mlp, L = t["width"], t["mlp"], t["layers"]
    rg = 1.0 / math.sqrt(2.0 * L)
    for i in range(L):
        p = f"{prefix}transformer.resblocks.{i}."
        sd[p + "ln_1.weight"] = _vec(g, w, 0.1, 1.0)
        sd[p + "ln_1.bias"] = _vec(g, w)
        sd[p + "attn.in_proj_weight"] = _lin(g, 3 * w, w, 1.5)
        sd[p + "attn.in_proj_bias"] = _vec(g, 3 * w)
        sd[p + "attn.out_proj.weight"] = _lin(g, w, w, rg)
        sd[p + "attn.out_proj.bias"] = _vec(g, w)
        sd[p + "ln_2.weight"] = _vec(g, w, 0.1, 1.0)
        sd[p + "ln_2.bias"] = _vec(g, w)
        sd[p + "mlp.c_fc.weight"] = _lin(g, mlp, w)
        sd[p + "mlp.c_fc.bias"] = _vec(g, mlp)
        sd[p + "mlp.c_proj.weight"] = _lin(g, w, mlp, rg)
        sd[p + "mlp.c_proj.bias"] = _vec(g, w)


def random_clip_weights(arch: dict, seed: int = 1234) -> Dict[str, np.ndarray]:
    g = _rng(seed)
    sd: Dict[str, np.ndarray] = {}
    v, t, E = arch.get("vision"), arch.get("text"), arch["embed_dim"]
    if v:
        w, p = v["width"], v["patch"]
        grid = v.get("image_size", 224) // p
        sd["visual.conv1.weight"] = g.standard_normal((w, 3, p, p), dtype=np.float32) / np.float32(math.sqrt(3 * p * p))
        sd["visual.class_embedding"] = _vec(g, w, 0.5)
        sd["visual.positional_embedding"] = 0.5 * g.standard_normal((grid * grid + 1, w), dtype=np.float32)
        sd["visual.ln_pre.weight"] = _vec(g, w, 0.1, 1.0)
        sd["visual.ln_pre.bias"] = _vec(g, w)
        _clip_blocks(g, "visual.", v, sd)
        sd["visual.ln_post.weight"] = _vec(g, w, 0.1, 1.0)
        sd["visual.ln_post.bias"] = _vec(g, w)
        sd["visual.proj"] = g.standard_normal((w, E), dtype=np.float32) / np.float32(math.sqrt(w))
    if t:
        w = t["width"]
        sd["token_embedding.weight"] = g.standard_normal((t["vocab"], w), dtype=np.float32)
        sd["positional_embedding"] = 0.5 * g.standard_normal((t["ctx"], w), dtype=np.float32)
        _clip_blocks(g, "", t, sd)
        sd["ln_final.weight"] = _vec(g, w, 0.1, 1.0)
        sd["ln_final.bias"] = _vec(g, w)
        sd["text_projection"] = g.standard_normal((w, E), dtype=np.float32) / np.float32(math.sqrt(w))
    return sd


def random_siglip_weights(arch: dict, seed: int = 1234) -> Dict[str, np.ndarray]:
    """Seeded random weights under open_clip's SigLIP state-dict names (timm trunk + open_clip text tower; arch: the
    registry's SigLIP block)."""
    g = _rng(seed)
    sd: Dict[str, np.ndarray] = {}
    v, t, E = arch.get("vision"), arch.get("text"), arch["embed_dim"]
    if v:
        w, p, mlp = v["width"], v["patch"], v["mlp"]
        grid = v["image_size"] // p
        rg = 1.0 / math.sqrt(2.0 * v["layers"])
        tr = "visual.trunk."
        sd[tr + "patch_embed.proj.weight"] = g.standard_normal((w, 3, p, p), dtype=np.float32) / np.float32(
            math.sqrt(3 * p * p))
        sd[tr + "patch_embed.proj.bias"] = _vec(g, w)
        sd[tr + "pos_embed"] = 0.5 * g.standard_normal((1, grid * grid, w), dtype=np.float32)
        for i in range(v["layers"]):
            b = f"{tr}blocks.{i}."
            sd[b + "norm1.weight"] = _vec(g, w, 0.1, 1.0)
            sd[b + "norm1.bias"] = _vec(g, w)
            sd[b + "attn.qkv.weight"] = _lin(g, 3 * w, w, 1.5)
            sd[b + "attn.qkv.bias"] = _vec(g, 3 * w)
            sd[b + "attn.proj.weight"] = _lin(g, w, w, rg)
            sd[b + "attn.proj.bias"] = _vec(g, w)
            sd[b + "norm2.weight"] = _vec(g, w, 0.1, 1.0)
            sd[b + "norm2.bias"] = _vec(g, w)
            sd[b + "mlp.fc1.weight"] = _lin(g, mlp, w)
            sd[b + "mlp.fc1.bias"] = _vec(g, mlp)
            sd[b + "mlp.fc2.weight"] = _lin(g, w, mlp, rg)
            sd[b + "mlp.fc2.bias"] = _vec(g, w)
        sd[tr + "norm.weight"] = _vec(g, w, 0.1, 1.0)
        sd[tr + "norm.bias"] = _vec(g, w)
        a, hm = tr + "attn_pool.", v.get("map_mlp", 4 * w)
        sd[a + "latent"] = g.standard_normal((1, 1, w), dtype=np.float32)
        sd[a + "q.weight"] = _lin(g, w, w, 1.5)
        sd[a + "q.bias"] = _vec(g, w)
        sd[a + "kv.weight"] = _lin(g, 2 * w, w, 1.5)
        sd[a + "kv.bias"] = _vec(g, 2 * w)
        sd[a + "proj.weight"] = _lin(g, w, w)
        sd[a + "proj.bias"] = _vec(g, w)
        sd[a + "norm.weight"] = _vec(g, w, 0.1, 1.0)
        sd[a + "norm.bias"] = _vec(g, w)
        sd[a + "mlp.fc1.weight"] = _lin(g, hm, w)
        sd[a + "mlp.fc1.bias"] = _vec(g, hm)
        sd[a + "mlp.fc2.weight"] = _lin(g, w, hm)
        sd[a + "mlp.fc2.bias"] = _vec(g, w)
    if t:
        w = t["width"]
        sd["text.token_embedding.weight"] = g.standard_normal((t["vocab"], w), dtype=np.float32)
        sd["text.positional_embedding"] = 0.5 * g.standard_normal((t["ctx"], w), dtype=np.float32)
        _clip_blocks(g, "text.", t, sd)
        sd["text.ln_final.weight"] = _vec(g, w, 0.1, 1.0)
        sd["text.ln_final.bias"] = _vec(g, w)
        sd["text.text_projection.weight"] = _lin(g, E, w)
        sd["text.text_projection.bias"] = _vec(g, E)
    return sd


def _bn(g, prefix, c, sd):
    sd[prefix + ".weight"] = _vec(g, c, 0.1, 1.0)
    sd[prefix + ".bias"] = _vec(g, c)
    sd[prefix + ".running_mean"] = _vec(g, c)
    sd[prefix + ".running_var"] = (0.5 + g.random(c, dtype=np.float32)).astype(np.float32)


def _conv(g, cout, cin, k):
    return g.standard_normal((cout, cin, k, k), dtype=np.float32) / np.float32(math.sqrt(cin * k * k))


def random_clip_resnet_weights(arch: dict, seed: int = 1234) -> Dict[str, np.ndarray]:
    """Seeded random weights under open_clip's ModifiedResNet CLIP names (arch: the registry's clip_resnet block;
    arch["resnet"] None: no image tower, arch["layers"] 0: no text tower)."""
    g = _rng(seed)
    sd: Dict[str, np.ndarray] = {}
    r, E = arch.get("resnet"), arch["embed_dim"]
    if r:
        w, v = r["width"], "visual."
        for i, (cin, cout) in enumerate(((3, w // 2), (w // 2, w // 2), (w // 2, w)), start=1):
            sd[f"{v}conv{i}.weight"] = _conv(g, cout, cin, 3)
            _bn(g, f"{v}bn{i}", cout, sd)
        inplanes = w
        for s, depth in enumerate(r["layers"]):
            planes = w << s
            for i in range(depth):
                p = f"{v}layer{s + 1}.{i}."
                for j, (cin, cout, k) in enumerate(((inplanes, planes, 1), (planes, planes, 3), (planes, 4 * planes, 1)),
                                                   start=1):
                    sd[f"{p}conv{j}.weight"] = _conv(g, cout, cin, k)
                    _bn(g, f"{p}bn{j}", cout, sd)
                if i == 0:   # stride 2 (stages 2-4) or 64 -> 256 channels (stage 1): a downsample branch
                    sd[f"{p}downsample.0.weight"] = _conv(g, 4 * planes, inplanes, 1)
                    _bn(g, f"{p}downsample.1", 4 * planes, sd)
                inplanes = 4 * planes
        C, grid = 32 * w, r.get("image_size", 224) // 32
        a = f"{v}attnpool."
        sd[a + "positional_embedding"] = g.standard_normal((grid * grid + 1, C), dtype=np.float32) / np.float32(
            math.sqrt(C))
        for nm, out_f in (("q_proj", C), ("k_proj", C), ("v_proj", C), ("c_proj", E)):
            sd[f"{a}{nm}.weight"] = _lin(g, out_f, C)
            sd[f"{a}{nm}.bias"] = _vec(g, out_f)
    if arch.get("layers"):
        t = {k: arch[k] for k in ("width", "layers", "heads", "mlp", "ctx", "vocab")}
        text = random_clip_weights({"embed_dim": E, "text": t}, seed + 1)
        sd.update(text)
    return sd


def random_clip_convnext_weights(arch: dict, seed: int = 1234) -> Dict[str, np.ndarray]:
    """Seeded random weights under open_clip's TimmModel names for a timm ConvNeXt trunk (arch: the registry's
    clip_convnext block; arch["convnext"] None: no image tower, arch["layers"] 0: no text tower)."""
    g = _rng(seed)
    sd: Dict[str, np.ndarray] = {}
    cx, E = arch.get("convnext"), arch["embed_dim"]
    if cx:
        t, dims = "visual.trunk.", cx["dims"]

        def ln(prefix, c):
            sd[prefix + ".weight"] = _vec(g, c, 0.1, 1.0)
            sd[prefix + ".bias"] = _vec(g, c)

        sd[t + "stem.0.weight"] = _conv(g, dims[0], 3, 4)
        sd[t + "stem.0.bias"] = _vec(g, dims[0])
        ln(t + "stem.1", dims[0])
        for s, (C, depth) in enumerate(zip(dims, cx["depths"])):
            p = f"{t}stages.{s}."
            if s > 0:
                ln(p + "downsample.0", dims[s - 1])
                sd[p + "downsample.1.weight"] = _conv(g, C, dims[s - 1], 2)
                sd[p + "downsample.1.bias"] = _vec(g, C)
            for i in range(depth):
                b = f"{p}blocks.{i}."
                sd[b + "conv_dw.weight"] = _conv(g, C, 1, 7)
                sd[b + "conv_dw.bias"] = _vec(g, C)
                ln(b + "norm", C)
                sd[b + "mlp.fc1.weight"] = _lin(g, 4 * C, C)
                sd[b + "mlp.fc1.bias"] = _vec(g, 4 * C)
                sd[b + "mlp.fc2.weight"] = _lin(g, C, 4 * C)
                sd[b + "mlp.fc2.bias"] = _vec(g, C)
                # trained layer scales are small; these keep the residual stream from growing over 30 blocks
                sd[b + "gamma"] = _vec(g, C, 0.1, 0.3)
        ln(t + "head.norm", dims[3])
        if cx["head"] == "mlp":
            sd["visual.head.mlp.fc1.weight"] = _lin(g, 2 * E, dims[3])
            sd["visual.head.mlp.fc1.bias"] = _vec(g, 2 * E)
            sd["visual.head.mlp.fc2.weight"] = _lin(g, E, 2 * E)
        else:
            sd["visual.head.proj.weight"] = _lin(g, E, dims[3])
    if arch.get("layers"):
        text = {k: arch[k] for k in ("width", "layers", "heads", "mlp", "ctx", "vocab")}
        sd.update(random_clip_weights({"embed_dim": E, "text": text}, seed + 1))
    return sd


def random_eva02_weights(arch: dict, seed: int = 1234) -> Dict[str, np.ndarray]:
    """Seeded random weights under open_clip's CustomTextCLIP names over a timm Eva trunk (arch: the registry's
    clip_eva block; arch["eva"] None: no image tower, arch["layers"] 0: no text tower)."""
    g = _rng(seed)
    sd: Dict[str, np.ndarray] = {}
    ev, E = arch.get("eva"), arch["embed_dim"]
    if ev:
        w, p, hid, L = ev["width"], ev["patch"], ev["mlp"], ev["layers"]
        grid = ev["image_size"] // p
        rg = 1.0 / math.sqrt(2.0 * L)
        tr = "visual.trunk."

        def ln(prefix, n):
            sd[prefix + ".weight"] = _vec(g, n, 0.1, 1.0)
            sd[prefix + ".bias"] = _vec(g, n)

        sd[tr + "patch_embed.proj.weight"] = _conv(g, w, 3, p)
        sd[tr + "patch_embed.proj.bias"] = _vec(g, w)
        sd[tr + "cls_token"] = 0.5 * g.standard_normal((1, 1, w), dtype=np.float32)
        sd[tr + "pos_embed"] = 0.5 * g.standard_normal((1, grid * grid + 1, w), dtype=np.float32)
        for i in range(L):
            b = f"{tr}blocks.{i}."
            ln(b + "norm1", w)
            sd[b + "attn.q_proj.weight"] = _lin(g, w, w, 1.5)
            sd[b + "attn.q_proj.bias"] = _vec(g, w)
            sd[b + "attn.k_proj.weight"] = _lin(g, w, w, 1.5)
            sd[b + "attn.v_proj.weight"] = _lin(g, w, w, 1.5)
            sd[b + "attn.v_proj.bias"] = _vec(g, w)
            ln(b + "attn.norm", w)
            sd[b + "attn.proj.weight"] = _lin(g, w, w, rg)
            sd[b + "attn.proj.bias"] = _vec(g, w)
            ln(b + "norm2", w)
            sd[b + "mlp.fc1_g.weight"] = _lin(g, hid, w)
            sd[b + "mlp.fc1_g.bias"] = _vec(g, hid)
            sd[b + "mlp.fc1_x.weight"] = _lin(g, hid, w)
            sd[b + "mlp.fc1_x.bias"] = _vec(g, hid)
            ln(b + "mlp.norm", hid)
            sd[b + "mlp.fc2.weight"] = _lin(g, w, hid, rg)
            sd[b + "mlp.fc2.bias"] = _vec(g, w)
        ln(tr + "norm", w)
        sd[tr + "head.weight"] = _lin(g, E, w)
        sd[tr + "head.bias"] = _vec(g, E)
    if arch.get("layers"):
        t = {k: arch[k] for k in ("width", "layers", "heads", "mlp", "ctx", "vocab")}
        text = random_clip_weights({"embed_dim": E, "text": t}, seed + 1)
        sd.update({"text." + k: v for k, v in text.items()})
    return sd


def random_bert_weights(arch: dict, seed: int = 1234) -> Dict[str, np.ndarray]:
    g = _rng(seed)
    w, mlp = arch["width"], arch["mlp"]
    sd: Dict[str, np.ndarray] = {}
    sd["embeddings.word_embeddings.weight"] = g.standard_normal((arch["vocab"], w), dtype=np.float32)
    sd["embeddings.position_embeddings.weight"] = 0.5 * g.standard_normal((arch.get("max_pos", 512), w), dtype=np.float32)
    sd["embeddings.token_type_embeddings.weight"] = 0.5 * g.standard_normal((arch.get("type_vocab", 2), w), dtype=np.float32)
    sd["embeddings.LayerNorm.weight"] = _vec(g, w, 0.1, 1.0)
    sd["embeddings.LayerNorm.bias"] = _vec(g, w)
    for i in range(arch["layers"]):
        p = f"encoder.layer.{i}."
        for nm in ("query", "key", "value"):
            sd[p + f"attention.self.{nm}.weight"] = _lin(g, w, w, 1.5)
            sd[p + f"attention.self.{nm}.bias"] = _vec(g, w)
        sd[p + "attention.output.dense.weight"] = _lin(g, w, w)
        sd[p + "attention.output.dense.bias"] = _vec(g, w)
        sd[p + "attention.output.LayerNorm.weight"] = _vec(g, w, 0.1, 1.0)
        sd[p + "attention.output.LayerNorm.bias"] = _vec(g, w)
        sd[p + "intermediate.dense.weight"] = _lin(g, mlp, w)
        sd[p + "intermediate.dense.bias"] = _vec(g, mlp)
        sd[p + "output.dense.weight"] = _lin(g, w, mlp)
        sd[p + "output.dense.bias"] = _vec(g, w)
        sd[p + "output.LayerNorm.weight"] = _vec(g, w, 0.1, 1.0)
        sd[p + "output.LayerNorm.bias"] = _vec(g, w)
    return sd


def random_xlmr_weights(arch: dict, seed: int = 1234) -> Dict[str, np.ndarray]:
    """Seeded random weights under HF XLMRobertaModel parameter names (arch: the registry's XLM-R block): BertModel's
    names with max_pos position rows and type_vocab (1) token-type rows."""
    return random_bert_weights(arch, seed)


def random_gte_weights(arch: dict, seed: int = 1234) -> Dict[str, np.ndarray]:
    """Seeded random weights under NewModel parameter names (arch: the registry's GTE block): the fused qkv_proj, the
    fused up_gate_proj [2 mlp, width] without bias, no position table.  up_gate_proj and down_proj have gains 0.7 and
    0.5: the GeGLU product of two Gaussian columns is heavier-tailed than a GELU's input, and at gain 1 the 24 post-LN
    layers amplify bf16 rounding to cosines near 0.99 against fp32 (trained checkpoints are not that sensitive)."""
    g = _rng(seed)
    w, mlp = arch["width"], arch["mlp"]
    sd: Dict[str, np.ndarray] = {}
    sd["embeddings.word_embeddings.weight"] = g.standard_normal((arch["vocab"], w), dtype=np.float32)
    sd["embeddings.token_type_embeddings.weight"] = 0.5 * g.standard_normal((arch.get("type_vocab", 2), w), dtype=np.float32)
    sd["embeddings.LayerNorm.weight"] = _vec(g, w, 0.1, 1.0)
    sd["embeddings.LayerNorm.bias"] = _vec(g, w)
    for i in range(arch["layers"]):
        p = f"encoder.layer.{i}."
        sd[p + "attention.qkv_proj.weight"] = _lin(g, 3 * w, w, 1.5)
        sd[p + "attention.qkv_proj.bias"] = _vec(g, 3 * w)
        sd[p + "attention.o_proj.weight"] = _lin(g, w, w)
        sd[p + "attention.o_proj.bias"] = _vec(g, w)
        sd[p + "attn_ln.weight"] = _vec(g, w, 0.1, 1.0)
        sd[p + "attn_ln.bias"] = _vec(g, w)
        sd[p + "mlp.up_gate_proj.weight"] = _lin(g, 2 * mlp, w, 0.7)
        sd[p + "mlp.down_proj.weight"] = _lin(g, w, mlp, 0.5)
        sd[p + "mlp.down_proj.bias"] = _vec(g, w)
        sd[p + "mlp_ln.weight"] = _vec(g, w, 0.1, 1.0)
        sd[p + "mlp_ln.bias"] = _vec(g, w)
    return sd


def random_mpnet_weights(arch: dict, seed: int = 1234) -> Dict[str, np.ndarray]:
    """Seeded random weights under HF MPNetModel parameter names (arch: the registry's MPNet block)."""
    g = _rng(seed)
    w, mlp = arch["width"], arch["mlp"]
    sd: Dict[str, np.ndarray] = {}
    sd["embeddings.word_embeddings.weight"] = g.standard_normal((arch["vocab"], w), dtype=np.float32)
    sd["embeddings.position_embeddings.weight"] = 0.5 * g.standard_normal((arch["max_pos"], w), dtype=np.float32)
    sd["embeddings.LayerNorm.weight"] = _vec(g, w, 0.1, 1.0)
    sd["embeddings.LayerNorm.bias"] = _vec(g, w)
    sd["encoder.relative_attention_bias.weight"] = _vec(g, arch.get("rel_buckets", 32) * arch["heads"], 1.0).reshape(
        -1, arch["heads"])
    for i in range(arch["layers"]):
        p = f"encoder.layer.{i}."
        for nm in ("q", "k", "v"):
            sd[p + f"attention.attn.{nm}.weight"] = _lin(g, w, w, 1.5)
            sd[p + f"attention.attn.{nm}.bias"] = _vec(g, w)
        sd[p + "attention.attn.o.weight"] = _lin(g, w, w)
        sd[p + "attention.attn.o.bias"] = _vec(g, w)
        sd[p + "attention.LayerNorm.weight"] = _vec(g, w, 0.1, 1.0)
        sd[p + "attention.LayerNorm.bias"] = _vec(g, w)
        sd[p + "intermediate.dense.weight"] = _lin(g, mlp, w)
        sd[p + "intermediate.dense.bias"] = _vec(g, mlp)
        sd[p + "output.dense.weight"] = _lin(g, w, mlp)
        sd[p + "output.dense.bias"] = _vec(g, w)
        sd[p + "output.LayerNorm.weight"] = _vec(g, w, 0.1, 1.0)
        sd[p + "output.LayerNorm.bias"] = _vec(g, w)
    return sd


def random_weights(kind: str, arch: dict, seed: int) -> Dict[str, np.ndarray]:
    """Seeded random weights for an Encoder of `kind` ("clip", "siglip", "clip_resnet", "clip_convnext", "clip_eva",
    "bert", "mpnet", "xlmr" or "gte"); KeyError for any other kind."""
    return {"clip": random_clip_weights, "siglip": random_siglip_weights, "clip_resnet": random_clip_resnet_weights,
            "clip_convnext": random_clip_convnext_weights, "clip_eva": random_eva02_weights,
            "bert": random_bert_weights, "mpnet": random_mpnet_weights, "xlmr": random_xlmr_weights,
            "gte": random_gte_weights}[kind](arch, seed)
