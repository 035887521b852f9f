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
    """.npz, torch .pt/.bin/.pth (a state dict or a TorchScript archive) or .safetensors -> {name: fp32 ndarray}."""
    p = str(path)
    if p.endswith(".npz"):
        with np.load(p) as z:
            return {k: np.asarray(z[k], dtype=np.float32) for k in z.files}
    if p.endswith(".safetensors"):
        from safetensors.numpy import load_file  # optional dependency
        return {k: np.asarray(v, dtype=np.float32) for k, v in load_file(p).items()}
    import torch
    if _is_torchscript(p):
        # OpenAI's released CLIP checkpoints (and open_clip's */openai files) are TorchScript archives, which
        # torch.load(weights_only=True) refuses; the scripted module's state dict has the names clip.load reads
        sd = torch.jit.load(p, map_location="cpu").state_dict()
    else:
        sd = torch.load(p, map_location="cpu", weights_only=True)
    if isinstance(sd, dict) and "state_dict" in sd and isinstance(sd["state_dict"], dict):
        sd = sd["state_dict"]
    out = {}
    for k, v in sd.items():
        if hasattr(v, "is_floating_point") and v.is_floating_point():
            out[k[len("module."):] if k.startswith("module.") else k] = v.float().numpy()
    return out


def _is_torchscript(path: str) -> bool:
    """A torch.jit.save archive: a zip whose records include the scripted code's constants.pkl (a plain torch.save
    zip has data.pkl only)."""
    import zipfile
    if not zipfile.is_zipfile(path):
        return False
    with zipfile.ZipFile(path) as z:
        return any(n.endswith("/constants.pkl") for n in z.namelist())


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
        pw = w
        if v.get("attn_pool_heads"):   # CoCa's attentional pooler: 256 queries of E columns attend over the tokens
            pw, a = E, "visual.attn_pool."
            sd[a + "query"] = g.standard_normal((256, E), dtype=np.float32)
            sd[a + "ln_q.weight"] = _vec(g, E, 0.1, 1.0)
            sd[a + "ln_q.bias"] = _vec(g, E)
            sd[a + "ln_k.weight"] = _vec(g, w, 0.1, 1.0)
            sd[a + "ln_k.bias"] = _vec(g, w)
            sd[a + "attn.q_proj_weight"] = _lin(g, E, E, 1.5)
            sd[a + "attn.k_proj_weight"] = _lin(g, E, w, 1.5)
            sd[a + "attn.v_proj_weight"] = _lin(g, E, w)
            sd[a + "attn.in_proj_bias"] = _vec(g, 3 * E)
            sd[a + "attn.out_proj.weight"] = _lin(g, E, E)
            sd[a + "attn.out_proj.bias"] = _vec(g, E)
        sd["visual.ln_post.weight"] = _vec(g, pw, 0.1, 1.0)
        sd["visual.ln_post.bias"] = _vec(g, pw)
        sd["visual.proj"] = g.standard_normal((pw, E), dtype=np.float32) / np.float32(math.sqrt(pw))
    if t:
        w = t["width"]
        # CoCa keeps its text tower under "text." and appends a learned CLS row (cls_emb)
        p = "text." if t.get("embed_cls") else ""
        sd[p + "token_embedding.weight"] = g.standard_normal((t["vocab"], w), dtype=np.float32)
        sd[p + "positional_embedding"] = 0.5 * g.standard_normal((t["ctx"], w), dtype=np.float32)
        if p:
            sd[p + "cls_emb"] = g.standard_normal(w, dtype=np.float32)
        _clip_blocks(g, p, t, sd)
        sd[p + "ln_final.weight"] = _vec(g, w, 0.1, 1.0)
        sd[p + "ln_final.bias"] = _vec(g, w)
        sd[p + "text_projection"] = g.standard_normal((w, E), dtype=np.float32) / np.float32(math.sqrt(w))
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


def random_cross_encoder_weights(arch: dict, seed: int = 1234) -> Dict[str, np.ndarray]:
    """Seeded random weights of a BERT cross-encoder under BertForSequenceClassification's names (arch: the registry's
    cross-encoder block): random_bert_weights under "bert.", the pooler and the classifier of num_labels rows."""
    w, labels = arch["width"], arch["num_labels"]
    sd = {"bert." + k: v for k, v in random_bert_weights(arch, seed).items()}
    g = _rng(seed + 1)
    sd["bert.pooler.dense.weight"] = _lin(g, w, w, 1.5)
    sd["bert.pooler.dense.bias"] = _vec(g, w)
    sd["classifier.weight"] = _lin(g, labels, w, 2.0)
    sd["classifier.bias"] = _vec(g, labels)
    return sd


# transformers' CLIP-style encoder layer names -> open_clip's (the engine's) below a tower's resblock prefix
_OWL_LAYER_NAMES = {"layer_norm1.": "ln_1.", "layer_norm2.": "ln_2.", "self_attn.out_proj.": "attn.out_proj.",
                    "mlp.fc1.": "mlp.c_fc.", "mlp.fc2.": "mlp.c_proj."}
# and LanguageBind's temporal sub-layer (languagebind/video/modeling_video.py:180-187), whose q | k | v go to
# temporal_attn.in_proj_* as self_attn's go to attn.in_proj_*
_TEMPORAL_LAYER_NAMES = {"temporal_layer_norm1.": "temporal_ln_1.", "temporal_attn.out_proj.": "temporal_attn.out_proj.",
                         "temporal_embedding": "temporal_embedding"}
# the two OWL-ViT tensors the detector never reads: the CLIP image projection and the contrastive temperature
OWLVIT_UNUSED = ("owlvit.visual_projection.weight", "owlvit.logit_scale")


def _hf_clip_tower_tensor(key: str, rest: str, dst: str, a: np.ndarray, out: dict, qkv: dict, what: str,
                          layer_names: dict, attns: dict) -> None:
    """One tensor of a transformers CLIP-style tower, `rest` its name below the tower's prefix, under the engine's
    names below `dst`: pre_layrnorm (also spelt pre_layernorm) -> ln_pre, post_layernorm -> ln_post, final_layer_norm
    -> ln_final, a layer's q / k / v parts of each attention in `attns` (its transformers prefix -> the engine's fused
    in_proj_ prefix) collected in qkv, its other parts renamed by layer_names.  Any other name raises KeyError."""
    for a_name, b_name in (("pre_layrnorm.", "ln_pre."), ("pre_layernorm.", "ln_pre."),
                           ("post_layernorm.", "ln_post."), ("final_layer_norm.", "ln_final.")):
        if rest.startswith(a_name):
            out[dst + b_name + rest[len(a_name):]] = a
            return
    if not rest.startswith("encoder.layers."):
        raise KeyError(f"{key}: not {what} parameter the engine knows")
    i, sub = rest[len("encoder.layers."):].split(".", 1)
    p = f"{dst}transformer.resblocks.{i}."
    for src, fused in attns.items():
        if sub.startswith(src) and sub[len(src):len(src) + 2] in ("q_", "k_", "v_"):
            qkv.setdefault(p + fused + sub.rsplit(".", 1)[1], {})[sub[len(src)]] = a
            return
    for a_name, b_name in layer_names.items():
        if sub.startswith(a_name):
            out[p + b_name + sub[len(a_name):]] = a
            return
    raise KeyError(f"{key}: not {what} parameter the engine knows")


def _stack_qkv(qkv: dict, out: dict) -> None:
    for name, parts in qkv.items():
        out[name] = np.concatenate([parts["q"], parts["k"], parts["v"]], axis=0)


def _f32(v) -> np.ndarray:
    return np.asarray(v.detach().cpu().numpy() if hasattr(v, "detach") else v, dtype=np.float32)


def owlvit_state_dict_to_engine(sd: Dict[str, np.ndarray]) -> Dict[str, np.ndarray]:
    """An OwlViTForObjectDetection state dict under the engine's CLIP names (b200_model_desc owl_detect): q | k | v of
    every layer stacked into in_proj_weight / in_proj_bias, text_projection.weight transposed to text_projection
    [width, E], pre_layrnorm (also spelt pre_layernorm) -> visual.ln_pre, post_layernorm -> visual.ln_post, and the
    detector's layer_norm.*, class_head.* and box_head.* kept as they are.  Every tensor is used but OWLVIT_UNUSED and
    the position_ids buffers; any other name raises KeyError."""
    sd = {k: v for k, v in sd.items() if not k.endswith("position_ids") and k not in OWLVIT_UNUSED}
    out: Dict[str, np.ndarray] = {}
    qkv: Dict[str, Dict[str, np.ndarray]] = {}
    towers = (("owlvit.vision_model.", "visual."), ("owlvit.text_model.", ""))
    fixed = {"owlvit.vision_model.embeddings.class_embedding": "visual.class_embedding",
             "owlvit.vision_model.embeddings.patch_embedding.weight": "visual.conv1.weight",
             "owlvit.vision_model.embeddings.position_embedding.weight": "visual.positional_embedding",
             "owlvit.text_model.embeddings.token_embedding.weight": "token_embedding.weight",
             "owlvit.text_model.embeddings.position_embedding.weight": "positional_embedding"}
    for k, v in sd.items():
        a = _f32(v)
        if k in fixed:
            out[fixed[k]] = a
        elif k == "owlvit.text_projection.weight":
            out["text_projection"] = np.ascontiguousarray(a.T)
        elif k.startswith(("layer_norm.", "class_head.", "box_head.")):
            out[k] = a
        else:
            for src, dst in towers:
                if k.startswith(src):
                    _hf_clip_tower_tensor(k, k[len(src):], dst, a, out, qkv, "an OwlViTForObjectDetection",
                                          _OWL_LAYER_NAMES, {"self_attn.": "attn.in_proj_"})
                    break
            else:
                raise KeyError(f"{k}: not an OwlViTForObjectDetection parameter the engine knows")
    _stack_qkv(qkv, out)
    return out


def languagebind_video_state_dict_to_engine(sd: Dict[str, np.ndarray]) -> Dict[str, np.ndarray]:
    """A LanguageBindVideo state dict (languagebind/video/modeling_video.py:842-873) under the engine's names
    (b200_model_desc video_frames): the CLIP renames of owlvit_state_dict_to_engine for both towers, plus each vision
    layer's temporal_embedding [1, T, W] -> [T, W], temporal_layer_norm1 -> temporal_ln_1 and temporal_attn's q | k | v
    stacked into temporal_attn.in_proj_*; visual_projection.weight [E, W] and text_projection.weight transposed to
    visual.proj and text_projection [W, E]; logit_scale as [1].  A Conv3d patch embedding [W, 3, tube, P, P] of tube 1
    (CLIPVisionEmbeddings3D) loses its tube axis; one of tube > 1 keeps it, and the engine refuses its size.  Every
    tensor is used but the position_ids buffers; any other name raises KeyError."""
    out: Dict[str, np.ndarray] = {}
    qkv: Dict[str, Dict[str, np.ndarray]] = {}
    towers = (("vision_model.", "visual."), ("text_model.", ""))
    fixed = {"vision_model.embeddings.class_embedding": "visual.class_embedding",
             "vision_model.embeddings.position_embedding.weight": "visual.positional_embedding",
             "text_model.embeddings.token_embedding.weight": "token_embedding.weight",
             "text_model.embeddings.position_embedding.weight": "positional_embedding"}
    layer_names = {**_OWL_LAYER_NAMES, **_TEMPORAL_LAYER_NAMES}
    attns = {"self_attn.": "attn.in_proj_", "temporal_attn.": "temporal_attn.in_proj_"}
    for k, v in sd.items():
        if k.endswith("position_ids"):
            continue
        a = _f32(v)
        if k in fixed:
            out[fixed[k]] = a
        elif k == "vision_model.embeddings.patch_embedding.weight":
            out["visual.conv1.weight"] = a[:, :, 0] if a.ndim == 5 and a.shape[2] == 1 else a
        elif k in ("visual_projection.weight", "text_projection.weight"):
            out["visual.proj" if k[0] == "v" else "text_projection"] = np.ascontiguousarray(a.T)
        elif k == "logit_scale":
            out[k] = a.reshape(1)
        else:
            for src, dst in towers:
                if k.startswith(src):
                    _hf_clip_tower_tensor(k, k[len(src):], dst, a, out, qkv, "a LanguageBindVideo", layer_names,
                                          attns)
                    break
            else:
                raise KeyError(f"{k}: not a LanguageBindVideo parameter the engine knows")
    for name in [n for n in out if n.endswith(".temporal_embedding")]:
        out[name] = out[name].reshape(-1, out[name].shape[-1])
    _stack_qkv(qkv, out)
    return out


def random_languagebind_video_weights(arch: dict, seed: int = 1234, form: str = "vl_new") -> Dict[str, np.ndarray]:
    """Seeded random weights of a LanguageBindVideo under its checkpoint's names and shapes (arch: the registry's
    LanguageBind block, the CLIP block of Encoder("clip") with video_frames T).  form "vl_new": CLIPVisionEmbeddings3D's
    class_embedding [T, W] and Conv3d patch_embedding [W, 3, 1, P, P]; "vl": CLIPVisionEmbeddings' [W] and
    [W, 3, P, P].  Every temporal_embedding is [1, T, W]; logit_scale a scalar near log(100)."""
    g = _rng(seed)
    v, t, E, T = arch["vision"], arch["text"], arch["embed_dim"], arch["video_frames"]
    sd: Dict[str, np.ndarray] = {}

    def attention(p, w, rg):
        for nm in ("q_proj", "k_proj", "v_proj"):
            sd[p + f"{nm}.weight"] = _lin(g, w, w, 1.5)
            sd[p + f"{nm}.bias"] = _vec(g, w)
        sd[p + "out_proj.weight"] = _lin(g, w, w, rg)
        sd[p + "out_proj.bias"] = _vec(g, w)

    def layers(prefix, tw, temporal):
        w, mlp, L = tw["width"], tw["mlp"], tw["layers"]
        rg = 1.0 / math.sqrt(2.0 * L)
        for i in range(L):
            p = f"{prefix}encoder.layers.{i}."
            for nm in ("layer_norm1", "layer_norm2"):
                sd[p + nm + ".weight"] = _vec(g, w, 0.1, 1.0)
                sd[p + nm + ".bias"] = _vec(g, w)
            attention(p + "self_attn.", w, rg)
            sd[p + "mlp.fc1.weight"] = _lin(g, mlp, w)
            sd[p + "mlp.fc1.bias"] = _vec(g, mlp)
            sd[p + "mlp.fc2.weight"] = _lin(g, w, mlp, rg)
            sd[p + "mlp.fc2.bias"] = _vec(g, w)
            if temporal:
                sd[p + "temporal_embedding"] = (g.standard_normal((1, T, w), dtype=np.float32) *
                                                np.float32(w ** -0.5))
                sd[p + "temporal_layer_norm1.weight"] = _vec(g, w, 0.1, 1.0)
                sd[p + "temporal_layer_norm1.bias"] = _vec(g, w)
                attention(p + "temporal_attn.", w, rg)

    w, p = v["width"], v["patch"]
    grid = v["image_size"] // p
    vm = "vision_model."
    conv = g.standard_normal((w, 3, p, p), dtype=np.float32) / np.float32(math.sqrt(3 * p * p))
    if form == "vl_new":
        sd[vm + "embeddings.class_embedding"] = np.stack([_vec(g, w, 0.5) for _ in range(T)])
        sd[vm + "embeddings.patch_embedding.weight"] = np.ascontiguousarray(conv[:, :, None])
    else:
        sd[vm + "embeddings.class_embedding"] = _vec(g, w, 0.5)
        sd[vm + "embeddings.patch_embedding.weight"] = conv
    sd[vm + "embeddings.position_embedding.weight"] = 0.5 * g.standard_normal((grid * grid + 1, w), dtype=np.float32)
    sd[vm + "pre_layrnorm.weight"] = _vec(g, w, 0.1, 1.0)
    sd[vm + "pre_layrnorm.bias"] = _vec(g, w)
    layers(vm, v, True)
    sd[vm + "post_layernorm.weight"] = _vec(g, w, 0.1, 1.0)
    sd[vm + "post_layernorm.bias"] = _vec(g, w)
    tw = t["width"]
    tm = "text_model."
    sd[tm + "embeddings.token_embedding.weight"] = g.standard_normal((t["vocab"], tw), dtype=np.float32)
    sd[tm + "embeddings.position_embedding.weight"] = 0.5 * g.standard_normal((t["ctx"], tw), dtype=np.float32)
    layers(tm, t, False)
    sd[tm + "final_layer_norm.weight"] = _vec(g, tw, 0.1, 1.0)
    sd[tm + "final_layer_norm.bias"] = _vec(g, tw)
    sd["visual_projection.weight"] = _lin(g, E, w)
    sd["text_projection.weight"] = _lin(g, E, tw)
    sd["logit_scale"] = np.array(4.6052, np.float32)
    return sd


def random_owlvit_weights(arch: dict, seed: int = 1234) -> Dict[str, np.ndarray]:
    """Seeded random weights of an OWL-ViT detector under OwlViTForObjectDetection's names (arch: the registry's
    OWL-ViT block, the CLIP block of Encoder("clip")), including the two tensors the detector does not read."""
    g = _rng(seed)
    v, t, E = arch["vision"], arch["text"], arch["embed_dim"]
    sd: Dict[str, np.ndarray] = {}

    def layers(prefix, tw):
        w, mlp, L = tw["width"], tw["mlp"], tw["layers"]
        rg = 1.0 / math.sqrt(2.0 * L)
        for i in range(L):
            p = f"{prefix}encoder.layers.{i}."
            for nm in ("layer_norm1", "layer_norm2"):
                sd[p + nm + ".weight"] = _vec(g, w, 0.1, 1.0)
                sd[p + nm + ".bias"] = _vec(g, w)
            for nm in ("q_proj", "k_proj", "v_proj"):
                sd[p + f"self_attn.{nm}.weight"] = _lin(g, w, w, 1.5)
                sd[p + f"self_attn.{nm}.bias"] = _vec(g, w)
            sd[p + "self_attn.out_proj.weight"] = _lin(g, w, w, rg)
            sd[p + "self_attn.out_proj.bias"] = _vec(g, w)
            sd[p + "mlp.fc1.weight"] = _lin(g, mlp, w)
            sd[p + "mlp.fc1.bias"] = _vec(g, mlp)
            sd[p + "mlp.fc2.weight"] = _lin(g, w, mlp, rg)
            sd[p + "mlp.fc2.bias"] = _vec(g, w)

    w, p = v["width"], v["patch"]
    grid = v["image_size"] // p
    vm = "owlvit.vision_model."
    sd[vm + "embeddings.class_embedding"] = _vec(g, w, 0.5)
    sd[vm + "embeddings.patch_embedding.weight"] = (g.standard_normal((w, 3, p, p), dtype=np.float32) /
                                                    np.float32(math.sqrt(3 * p * p)))
    sd[vm + "embeddings.position_embedding.weight"] = 0.5 * g.standard_normal((grid * grid + 1, w), dtype=np.float32)
    sd[vm + "pre_layrnorm.weight"] = _vec(g, w, 0.1, 1.0)
    sd[vm + "pre_layrnorm.bias"] = _vec(g, w)
    layers(vm, v)
    sd[vm + "post_layernorm.weight"] = _vec(g, w, 0.1, 1.0)
    sd[vm + "post_layernorm.bias"] = _vec(g, w)
    tw = t["width"]
    tm = "owlvit.text_model."
    sd[tm + "embeddings.token_embedding.weight"] = g.standard_normal((t["vocab"], tw), dtype=np.float32)
    sd[tm + "embeddings.position_embedding.weight"] = 0.5 * g.standard_normal((t["ctx"], tw), dtype=np.float32)
    layers(tm, t)
    sd[tm + "final_layer_norm.weight"] = _vec(g, tw, 0.1, 1.0)
    sd[tm + "final_layer_norm.bias"] = _vec(g, tw)
    sd["owlvit.text_projection.weight"] = _lin(g, E, tw)
    sd["owlvit.visual_projection.weight"] = _lin(g, E, w)
    sd["owlvit.logit_scale"] = np.array(2.6592, np.float32)
    sd["layer_norm.weight"] = _vec(g, w, 0.1, 1.0)
    sd["layer_norm.bias"] = _vec(g, w)
    sd["class_head.dense0.weight"] = _lin(g, E, w)
    sd["class_head.dense0.bias"] = _vec(g, E)
    # shift and scale spread around 0 so that both branches of the ELU occur among the patches
    sd["class_head.logit_shift.weight"] = _lin(g, 1, w)
    sd["class_head.logit_shift.bias"] = _vec(g, 1)
    sd["class_head.logit_scale.weight"] = _lin(g, 1, w)
    sd["class_head.logit_scale.bias"] = _vec(g, 1)
    for nm in ("dense0", "dense1"):
        sd[f"box_head.{nm}.weight"] = _lin(g, w, w)
        sd[f"box_head.{nm}.bias"] = _vec(g, w)
    sd["box_head.dense2.weight"] = _lin(g, 4, w)
    sd["box_head.dense2.bias"] = _vec(g, 4)
    return sd


def random_xlmr_weights(arch: dict, seed: int = 1234) -> Dict[str, np.ndarray]:
    """Seeded random weights under HF XLMRobertaModel parameter names (arch: the registry's XLM-R block): BertModel's
    names with max_pos position rows and type_vocab (1) token-type rows."""
    return random_bert_weights(arch, seed)


def random_mclip_text_weights(arch: dict, seed: int = 1234) -> Dict[str, np.ndarray]:
    """Seeded random weights of an M-CLIP text tower under MultilingualCLIP's names (arch: the registry's M-CLIP
    block): the BERT / XLM-R encoder under "transformer." and LinearTransformation [proj_dim, width] with its bias."""
    sd = {"transformer." + k: v for k, v in random_bert_weights(arch, seed).items()}
    g = _rng(seed + 1)
    sd["LinearTransformation.weight"] = _lin(g, arch["proj_dim"], arch["width"])
    sd["LinearTransformation.bias"] = _vec(g, arch["proj_dim"])
    return sd


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
