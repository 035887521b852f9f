"""ORACLE — TEST INFRASTRUCTURE ONLY.  CPU fp32 restatement of the XLM-RoBERTa forward the reference calls into for the
multilingual-e5 checkpoints, built on the BERT restatement of oracle/encoders.py.

The reference loads intfloat/multilingual-e5-{base,large,large-instruct} as `AutoModel` -> `XLMRobertaModel` and
mean-pools + L2-normalises its last hidden state (src/marqo/core/inference/embedding_models/hugging_face_model.py:
172-214).  Read from transformers 5.5.0 (modeling_xlm_roberta.py), XLMRobertaModel is BertModel except for its
embeddings:
  * position_ids = cumsum(ids != pad) * (ids != pad) + pad (create_position_ids_from_input_ids): from the ids, not the
    mask, so a row's pads take the pad row and its tokens count from pad + 1
  * one token-type row (type_vocab_size 1), LayerNorm eps 1e-5
`xlmr_encode` feeds oracle.encoders.bert_encode a per-call word table holding word[ids] + position[p] for every token
slot, a zero position table and slot indices as ids: the layers, the token-type row, pooling and normalisation are then
exactly the BERT restatement's.  Tested against transformers.XLMRobertaModel itself (tests/test_xlmr.py)."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Optional

import numpy as np
import torch

from oracle.encoders import BertCfg, bert_encode


@dataclass
class XlmrCfg:
    width: int = 768
    layers: int = 12
    heads: int = 12
    mlp: int = 3072
    vocab: int = 250002
    max_pos: int = 514          # max_position_embeddings: positions start after pad_id, so ctx = 512
    pad_id: int = 1
    type_vocab: int = 1
    ln_eps: float = 1e-5
    pool: str = "mean"


XLMR_BASE = XlmrCfg()
XLMR_LARGE = XlmrCfg(width=1024, layers=24, heads=16, mlp=4096)


def tiny_xlmr() -> XlmrCfg:
    return XlmrCfg(width=128, layers=2, heads=2, mlp=512, vocab=1000)


def engine_config(cfg: XlmrCfg) -> dict:
    """The Encoder("xlmr", ...) config (and registry arch block) of `cfg`."""
    return dict(kind="xlmr", width=cfg.width, layers=cfg.layers, heads=cfg.heads, mlp=cfg.mlp, vocab=cfg.vocab,
                max_pos=cfg.max_pos, pad_id=cfg.pad_id, type_vocab=cfg.type_vocab, ln_eps=cfg.ln_eps, pool=cfg.pool)


def make_xlmr_weights(cfg: XlmrCfg, seed: int = 1234) -> Dict[str, torch.Tensor]:
    """The engine's seeded XLM-R weights (marqo_b200.weights.random_xlmr_weights) as torch tensors."""
    from marqo_b200.weights import random_xlmr_weights
    return {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in random_xlmr_weights(engine_config(cfg), seed).items()}


def position_ids(ids: torch.Tensor, pad: int) -> torch.Tensor:
    keep = (ids != pad).long()
    return torch.cumsum(keep, dim=1) * keep + pad


@torch.no_grad()
def xlmr_encode(sd, cfg: XlmrCfg, ids: torch.Tensor, attn_mask: Optional[torch.Tensor] = None,
                normalize: bool = True) -> torch.Tensor:
    """XLMRobertaModel forward (eval) + Marqo's pooling / F.normalize (hugging_face_model.py:188-214)."""
    ids = ids.long()
    B, S = ids.shape
    w = cfg.width
    slots = (sd["embeddings.word_embeddings.weight"][ids]
             + sd["embeddings.position_embeddings.weight"][position_ids(ids, cfg.pad_id)])
    flat = dict(sd)
    flat["embeddings.word_embeddings.weight"] = slots.reshape(B * S, w)
    flat["embeddings.position_embeddings.weight"] = torch.zeros(S, w)
    bcfg = BertCfg(cfg.width, cfg.layers, cfg.heads, cfg.mlp, vocab=B * S, max_pos=S, type_vocab=cfg.type_vocab,
                   pool=cfg.pool, ln_eps=cfg.ln_eps)
    return bert_encode(flat, bcfg, torch.arange(B * S).view(B, S), attn_mask, normalize)


def hf_config(cfg: XlmrCfg):
    """transformers.XLMRobertaConfig of `cfg` (eager attention, no dropout)."""
    from transformers import XLMRobertaConfig
    return XLMRobertaConfig(vocab_size=cfg.vocab, hidden_size=cfg.width, num_hidden_layers=cfg.layers,
                            num_attention_heads=cfg.heads, intermediate_size=cfg.mlp,
                            max_position_embeddings=cfg.max_pos, type_vocab_size=cfg.type_vocab,
                            pad_token_id=cfg.pad_id, bos_token_id=0, eos_token_id=2, layer_norm_eps=cfg.ln_eps,
                            hidden_act="gelu", hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0,
                            attn_implementation="eager")


def fairseq_ids(sp, text: str) -> list:
    """XLMRobertaTokenizer's ids from a sentencepiece.SentencePieceProcessor: <s> spm ids + 1 (<unk> -> 3) </s>."""
    return [0] + [3 if i == sp.unk_id() else i + 1 for i in sp.encode(text)] + [2]


def ragged_ids(g: torch.Generator, B: int, S: int, lens, vocab: int, pad: int = 1):
    """Right-padded rows "<s> ... </s>" of the given lengths with random ids in [4, vocab), and their masks."""
    ids = torch.randint(4, vocab, (B, S), generator=g)
    ids[:, 0] = 0
    mask = torch.ones(B, S, dtype=torch.int64)
    for b in range(B):
        L = int(lens[b])
        ids[b, L - 1] = 2
        ids[b, L:] = pad
        mask[b, L:] = 0
    return ids, mask
