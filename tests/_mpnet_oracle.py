"""ORACLE — TEST INFRASTRUCTURE ONLY.  CPU fp32 restatement of the MPNet forward the reference calls into, beside the
CLIP / BERT restatements of oracle/encoders.py.

The reference loads the sentence-transformers MPNet checkpoints (hf/all-mpnet-base-v1/v2, hf/all_datasets_v3/v4_mpnet-
base) as `AutoModel` -> `MPNetModel` and mean-pools + L2-normalises its last hidden state
(src/marqo/core/inference/embedding_models/hugging_face_model.py:172-214).  The arithmetic below is read from
transformers 5.5.0 (modeling_mpnet.py); the reference pins transformers 4.41.2, which cannot be read offline:
  * embeddings: word_embeddings[ids] + position_embeddings[position_ids], LayerNorm; no token types; position_ids =
    cumsum(ids != pad) * (ids != pad) + pad (create_position_ids_from_input_ids) — from the ids, not the mask
  * one relative-position bias table [buckets, heads] shared by every layer: bias[h, i, j] = table[bucket(j - i), h]
    with token indices i (query), j (key) (MPNetEncoder.compute_position_bias, relative_position_bucket)
  * post-LN layers: LN(o(softmax(q k^T / sqrt(hd) + bias + key mask) v) + x), LN(W2 GELU_erf(W1 x) + x)
Tested against transformers.MPNetModel itself (tests/test_mpnet.py)."""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional

import torch
import torch.nn.functional as F


@dataclass
class MpnetCfg:
    width: int = 768
    layers: int = 12
    heads: int = 12
    mlp: int = 3072
    vocab: int = 30527
    max_pos: int = 514          # max_position_embeddings
    pad_id: int = 1
    ln_eps: float = 1e-5
    rel_buckets: int = 32
    rel_max_distance: int = 128
    pool: str = "mean"


MPNET_BASE = MpnetCfg()


def tiny_mpnet() -> MpnetCfg:
    return MpnetCfg(width=128, layers=2, heads=2, mlp=512, vocab=1000, max_pos=66)


def make_mpnet_weights(cfg: MpnetCfg, seed: int = 1234) -> Dict[str, torch.Tensor]:
    """Seeded O(1)-activation random weights under HF MPNetModel parameter names."""
    g = torch.Generator().manual_seed(seed)
    w = cfg.width

    def lin(out_f, in_f, gain=1.0):
        return torch.randn(out_f, in_f, generator=g) * (gain / math.sqrt(in_f))

    def vec(n, std=0.1, mean=0.0):
        return mean + std * torch.randn(n, generator=g)

    sd: Dict[str, torch.Tensor] = {}
    sd["embeddings.word_embeddings.weight"] = torch.randn(cfg.vocab, w, generator=g)
    sd["embeddings.position_embeddings.weight"] = 0.5 * torch.randn(cfg.max_pos, w, generator=g)
    sd["embeddings.LayerNorm.weight"] = vec(w, 0.1, 1.0)
    sd["embeddings.LayerNorm.bias"] = vec(w)
    sd["encoder.relative_attention_bias.weight"] = torch.randn(cfg.rel_buckets, cfg.heads, generator=g)
    for i in range(cfg.layers):
        p = f"encoder.layer.{i}."
        for nm in ("q", "k", "v"):
            sd[p + f"attention.attn.{nm}.weight"] = lin(w, w, 1.5)
            sd[p + f"attention.attn.{nm}.bias"] = vec(w)
        sd[p + "attention.attn.o.weight"] = lin(w, w)
        sd[p + "attention.attn.o.bias"] = vec(w)
        sd[p + "attention.LayerNorm.weight"] = vec(w, 0.1, 1.0)
        sd[p + "attention.LayerNorm.bias"] = vec(w)
        sd[p + "intermediate.dense.weight"] = lin(cfg.mlp, w)
        sd[p + "intermediate.dense.bias"] = vec(cfg.mlp)
        sd[p + "output.dense.weight"] = lin(w, cfg.mlp)
        sd[p + "output.dense.bias"] = vec(w)
        sd[p + "output.LayerNorm.weight"] = vec(w, 0.1, 1.0)
        sd[p + "output.LayerNorm.bias"] = vec(w)
    return sd


def relative_position_bucket(rel: torch.Tensor, num_buckets: int = 32, max_distance: int = 128) -> torch.Tensor:
    """Bucket of relative_position = key - query: n = -rel; keys after the query take the upper half; |n| < half / 2 is
    exact, the rest log-spaced in fp32 up to max_distance (truncated toward zero) and clipped to half - 1."""
    half = num_buckets // 2
    max_exact = half // 2
    n = -rel.long()
    ret = (n < 0).long() * half
    n = n.abs()
    large = max_exact + (torch.log(n.float() / max_exact) / math.log(max_distance / max_exact)
                         * (half - max_exact)).long()
    large = large.clamp(max=half - 1)
    return ret + torch.where(n < max_exact, n, large)


def position_ids(ids: torch.Tensor, pad: int) -> torch.Tensor:
    keep = (ids != pad).long()
    return torch.cumsum(keep, dim=1) * keep + pad


@torch.no_grad()
def mpnet_encode(sd, cfg: MpnetCfg, ids: torch.Tensor, attn_mask: Optional[torch.Tensor] = None,
                 normalize: bool = True) -> torch.Tensor:
    """MPNetModel forward (eval) + Marqo's pooling / F.normalize (hugging_face_model.py:188-214)."""
    ids = ids.long()
    B, S = ids.shape
    if attn_mask is None:
        attn_mask = torch.ones(B, S, dtype=torch.long)
    attn_mask = attn_mask.long()
    w, hd = cfg.width, cfg.width // cfg.heads
    x = sd["embeddings.word_embeddings.weight"][ids] + sd["embeddings.position_embeddings.weight"][position_ids(ids, cfg.pad_id)]
    x = F.layer_norm(x, (w,), sd["embeddings.LayerNorm.weight"], sd["embeddings.LayerNorm.bias"], cfg.ln_eps)
    rel = torch.arange(S)[None, :] - torch.arange(S)[:, None]                     # key - query
    bucket = relative_position_bucket(rel, cfg.rel_buckets, cfg.rel_max_distance)
    bias = sd["encoder.relative_attention_bias.weight"][bucket].permute(2, 0, 1)[None]   # [1, H, S, S]
    add_mask = (1.0 - attn_mask[:, None, None, :].float()) * torch.finfo(torch.float32).min
    for i in range(cfg.layers):
        p = f"encoder.layer.{i}."
        q = F.linear(x, sd[p + "attention.attn.q.weight"], sd[p + "attention.attn.q.bias"])
        k = F.linear(x, sd[p + "attention.attn.k.weight"], sd[p + "attention.attn.k.bias"])
        v = F.linear(x, sd[p + "attention.attn.v.weight"], sd[p + "attention.attn.v.bias"])
        q = q.view(B, S, cfg.heads, hd).transpose(1, 2)
        k = k.view(B, S, cfg.heads, hd).transpose(1, 2)
        v = v.view(B, S, cfg.heads, hd).transpose(1, 2)
        att = (q @ k.transpose(-1, -2)) / math.sqrt(hd) + bias + add_mask
        o = (att.softmax(dim=-1) @ v).transpose(1, 2).reshape(B, S, w)
        o = F.linear(o, sd[p + "attention.attn.o.weight"], sd[p + "attention.attn.o.bias"])
        x = F.layer_norm(o + x, (w,), sd[p + "attention.LayerNorm.weight"], sd[p + "attention.LayerNorm.bias"], cfg.ln_eps)
        h = F.gelu(F.linear(x, sd[p + "intermediate.dense.weight"], sd[p + "intermediate.dense.bias"]))
        h = F.linear(h, sd[p + "output.dense.weight"], sd[p + "output.dense.bias"])
        x = F.layer_norm(h + x, (w,), sd[p + "output.LayerNorm.weight"], sd[p + "output.LayerNorm.bias"], cfg.ln_eps)
    if cfg.pool == "cls":
        emb = x[:, 0]
    else:
        last = x.masked_fill(~attn_mask[..., None].bool(), 0.0)
        emb = last.sum(dim=1) / attn_mask.sum(dim=1)[..., None]
    if normalize:
        emb = F.normalize(emb, p=2, dim=1)
    return emb


def hf_config(cfg: MpnetCfg):
    """transformers.MPNetConfig of `cfg` (eager attention, no dropout)."""
    from transformers import MPNetConfig
    return MPNetConfig(vocab_size=cfg.vocab, hidden_size=cfg.width, num_hidden_layers=cfg.layers,
                       num_attention_heads=cfg.heads, intermediate_size=cfg.mlp, max_position_embeddings=cfg.max_pos,
                       pad_token_id=cfg.pad_id, layer_norm_eps=cfg.ln_eps, relative_attention_num_buckets=cfg.rel_buckets,
                       hidden_act="gelu", hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0,
                       attn_implementation="eager")


def engine_config(cfg: MpnetCfg) -> dict:
    """The Encoder("mpnet", ...) config of `cfg`."""
    return dict(width=cfg.width, layers=cfg.layers, heads=cfg.heads, mlp=cfg.mlp, vocab=cfg.vocab, max_pos=cfg.max_pos,
                pad_id=cfg.pad_id, ln_eps=cfg.ln_eps, rel_buckets=cfg.rel_buckets, rel_max_distance=cfg.rel_max_distance,
                pool=cfg.pool)


def synthetic_vocab(n: int) -> list:
    """An MPNet-style vocab.txt of n lines: <s> <pad> </s> <unk> first, then BERT's specials, words, some '##' pieces and
    <mask> last (as in the real vocabulary)."""
    head = ["<s>", "<pad>", "</s>", "<unk>", "[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"]
    pieces = ["##" + c for c in "abcdefghijklmnopqrstuvwxyz0123456789"]
    letters = list("abcdefghijklmnopqrstuvwxyz0123456789") + list("!\"#$%&'()*+,-./:;<=>?@[\\]^_`{|}~")
    words = ["the", "cat", "sat", "on", "mat", "mask", "cls", "sep", "unk", "pad", "hello", "world", "un", "##able",
             "##ing", "play", "run"]
    body = head + letters + pieces + words
    body += [f"w{i}" for i in range(n - len(body) - 1)]
    return body + ["<mask>"]
