"""ORACLE — TEST INFRASTRUCTURE ONLY.  fp32 torch restatement of the forward pass the reference runs for the Stella
embedder Marqo/dunzhang-stella_en_400M_v5: Alibaba's NewModel (gte-v1.5 architecture, trust_remote_code) loaded with
use_memory_efficient_attention False and unpad_inputs False, then masked mean pooling and F.normalize
(src/marqo/core/inference/embedding_models/hugging_face_model.py:172-214).  NewModel's modeling.py cannot be re-read
offline; the restatement is model_registry's docstring (verify):
  x = LN_emb(word[ids] + token_type[0])                               no position table
  per layer (post-LN):  q | k | v = x Wqkv^T + bqkv;  q, k rotated by position (rotate_half, the NTK table below)
                        x = attn_ln(x + softmax(q k^T / 8 + key mask) v Wo^T + bo)
                        up | gate = x Wug^T;  x = mlp_ln(x + (GELU(gate) * up) Wd^T + bd)
  RoPE: pair j = 0..31 of a head (columns j, j + 32) turns by s f_j, f_j = (theta factor)^(-2j/64) / factor^(2/64).
The formula is written once here and once in the engine's table builder (kernels::rope_table_ntk).  Runs on the CPU or
on the GPU (the caller moves the weights)."""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional

import numpy as np
import torch
import torch.nn.functional as F

NAME = "Marqo/dunzhang-stella_en_400M_v5"


@dataclass
class GteCfg:
    width: int = 1024
    layers: int = 24
    heads: int = 16
    mlp: int = 4096
    vocab: int = 30528
    type_vocab: int = 2
    ctx: int = 512
    ln_eps: float = 1e-12
    rope_theta: float = 160000.0
    rope_ntk_factor: float = 2.0
    pool: str = "mean"


STELLA = GteCfg()


def tiny_gte() -> GteCfg:
    return GteCfg(width=128, layers=2, heads=2, mlp=256, vocab=1000, ctx=128)


def engine_config(cfg: GteCfg) -> dict:
    """The Encoder("gte", ...) config (and registry arch block) of `cfg`."""
    return dict(kind="gte", width=cfg.width, layers=cfg.layers, heads=cfg.heads, mlp=cfg.mlp, vocab=cfg.vocab,
                type_vocab=cfg.type_vocab, ctx=cfg.ctx, ln_eps=cfg.ln_eps, rope_theta=cfg.rope_theta,
                rope_ntk_factor=cfg.rope_ntk_factor, pool=cfg.pool)


def make_gte_weights(cfg: GteCfg, seed: int = 1234) -> Dict[str, torch.Tensor]:
    """The engine's seeded NewModel weights (marqo_b200.weights.random_gte_weights) as torch tensors."""
    from marqo_b200.weights import random_gte_weights
    return {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in random_gte_weights(engine_config(cfg), seed).items()}


def inv_freq(cfg: GteCfg) -> torch.Tensor:
    """f_j, j = 0..31, in fp64."""
    j = torch.arange(32, dtype=torch.float64)
    base = cfg.rope_theta * cfg.rope_ntk_factor
    return base ** (-2.0 * j / 64.0) / cfg.rope_ntk_factor ** (2.0 / 64.0)


def rope_angles(cfg: GteCfg, S: int) -> torch.Tensor:
    """[S, 32] fp64 angles s f_j."""
    return torch.arange(S, dtype=torch.float64)[:, None] * inv_freq(cfg)[None, :]


def rotate(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> torch.Tensor:
    """x [B, S, H, 64], cos / sin [S, 32]: (a, b) = (x[..., j], x[..., j + 32]) -> (a cos - b sin, b cos + a sin)."""
    a, b = x[..., :32], x[..., 32:]
    c, s = cos[None, :, None, :], sin[None, :, None, :]
    return torch.cat([a * c - b * s, b * c + a * s], dim=-1)


def layer(sd, p: str, cfg: GteCfg, x: torch.Tensor, keep: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor):
    """One NewLayer (eval) over x [B, S, W]; keep [B, S] bool marks the real tokens (keys)."""
    B, S, w = x.shape
    H = cfg.heads
    qkv = x @ sd[p + "attention.qkv_proj.weight"].t() + sd[p + "attention.qkv_proj.bias"]
    q, k, v = (t.reshape(B, S, H, 64) for t in qkv.split(w, dim=-1))
    q, k = rotate(q, cos, sin), rotate(k, cos, sin)
    scores = torch.einsum("bqhd,bkhd->bhqk", q, k) / math.sqrt(64)
    scores = scores.masked_fill(~keep[:, None, None, :], float("-inf"))
    o = torch.einsum("bhqk,bkhd->bqhd", scores.softmax(dim=-1), v).reshape(B, S, w)
    x = F.layer_norm(x + o @ sd[p + "attention.o_proj.weight"].t() + sd[p + "attention.o_proj.bias"], (w,),
                     sd[p + "attn_ln.weight"], sd[p + "attn_ln.bias"], cfg.ln_eps)
    up, gate = (x @ sd[p + "mlp.up_gate_proj.weight"].t()).split(cfg.mlp, dim=-1)
    down = (F.gelu(gate) * up) @ sd[p + "mlp.down_proj.weight"].t() + sd[p + "mlp.down_proj.bias"]
    return F.layer_norm(x + down, (w,), sd[p + "mlp_ln.weight"], sd[p + "mlp_ln.bias"], cfg.ln_eps)


@torch.no_grad()
def gte_encode(sd, cfg: GteCfg, ids: torch.Tensor, attn_mask: Optional[torch.Tensor] = None,
               normalize: bool = True) -> torch.Tensor:
    """NewModel forward (eval) + Marqo's pooling / F.normalize, on the device of the weights."""
    dev = sd["embeddings.word_embeddings.weight"].device
    ids = ids.long().to(dev)
    B, S = ids.shape
    mask = torch.ones(B, S, dtype=torch.long, device=dev) if attn_mask is None else attn_mask.long().to(dev)
    w = cfg.width
    x = sd["embeddings.word_embeddings.weight"][ids] + sd["embeddings.token_type_embeddings.weight"][0]
    x = F.layer_norm(x, (w,), sd["embeddings.LayerNorm.weight"], sd["embeddings.LayerNorm.bias"], cfg.ln_eps)
    th = rope_angles(cfg, S).to(dev)
    cos, sin = th.cos().float(), th.sin().float()
    keep = mask.bool()
    for i in range(cfg.layers):
        x = layer(sd, f"encoder.layer.{i}.", cfg, x, keep, cos, sin)
    if cfg.pool == "cls":
        emb = x[:, 0]
    else:
        m = mask[..., None].to(x.dtype)
        emb = (x * m).sum(dim=1) / m.sum(dim=1)
    return F.normalize(emb, p=2, dim=1) if normalize else emb


def ragged_ids(g: torch.Generator, lens, S: int, vocab: int):
    """Right-padded rows "[CLS] ... [SEP]" (101, 102, pad 0) of the given lengths with random ids in [103, vocab),
    and their masks.  A row of length 1 is a lone [CLS]."""
    B = len(lens)
    ids = torch.randint(103, vocab, (B, S), generator=g)
    mask = torch.ones(B, S, dtype=torch.int64)
    for b, L in enumerate(lens):
        ids[b, 0] = 101
        if L > 1:
            ids[b, L - 1] = 102
        ids[b, L:] = 0
        mask[b, L:] = 0
    return ids, mask
