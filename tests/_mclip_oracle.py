"""ORACLE — TEST INFRASTRUCTURE ONLY.  CPU fp32 restatement of M-CLIP's text forward, the one the reference's
MULTILINGUAL_CLIP.encode_text calls (pt_multilingual_clip MultilingualCLIP.forward, verify; clip_utils.py:555-570):

    tok  = tokenizer(texts, padding=True)                     # no truncation
    embs = transformer(**tok)[0]                              # XLMRobertaModel or BertModel, last hidden state
    embs = (embs * mask[..., None]).sum(1) / mask.sum(1)[:, None]
    out  = LinearTransformation(embs)                         # nn.Linear(width, proj_dim), with bias
    out  = out / out.norm(dim=-1, keepdim=True)               # when normalize is set (no epsilon)

built on the XLM-R and BERT restatements (tests/_xlmr_oracle.py, oracle/encoders.py), whose masked mean it reuses.
Tested against transformers' XLMRobertaModel / BertModel and a torch Linear (tests/test_multilingual_clip.py)."""
from __future__ import annotations

import copy
from typing import Dict, Optional

import numpy as np
import torch

import _xlmr_oracle as X
from oracle.encoders import BertCfg, bert_encode

PREFIX = "transformer."


def arch(name: str, **edits) -> dict:
    """The registry arch of M-CLIP model `name` with the given top-level fields changed (layers=2, vocab=1000, ...)."""
    from marqo_b200 import model_registry as R
    a = copy.deepcopy(R.MULTILINGUAL_CLIP_MODELS[name]["arch"])
    a.update(edits)
    return a


def text_weights(a: dict, seed: int) -> Dict[str, torch.Tensor]:
    """The engine's seeded M-CLIP text weights (marqo_b200.weights.random_mclip_text_weights) as torch tensors."""
    from marqo_b200.weights import random_mclip_text_weights
    return {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in random_mclip_text_weights(a, seed).items()}


def _encoder_cfg(a: dict):
    if a["text_kind"] == "xlmr":
        return X.XlmrCfg(width=a["width"], layers=a["layers"], heads=a["heads"], mlp=a["mlp"], vocab=a["vocab"],
                         max_pos=a["max_pos"], pad_id=a["pad_id"], type_vocab=a["type_vocab"], ln_eps=a["ln_eps"])
    return BertCfg(a["width"], a["layers"], a["heads"], a["mlp"], vocab=a["vocab"], max_pos=a["max_pos"],
                   type_vocab=a["type_vocab"], ln_eps=a["ln_eps"])


@torch.no_grad()
def masked_mean(sd, a: dict, ids: torch.Tensor, mask: Optional[torch.Tensor]) -> torch.Tensor:
    """The encoder's last hidden state, mean-pooled over each row's tokens: fp32 [n, width]."""
    enc = {k[len(PREFIX):]: v for k, v in sd.items() if k.startswith(PREFIX)}
    cfg = _encoder_cfg(a)
    if a["text_kind"] == "xlmr":
        return X.xlmr_encode(enc, cfg, ids, mask, normalize=False)
    return bert_encode(enc, cfg, ids, mask, normalize=False)


@torch.no_grad()
def encode_text(sd, a: dict, ids: torch.Tensor, mask: Optional[torch.Tensor] = None,
                normalize: bool = True) -> torch.Tensor:
    out = masked_mean(sd, a, ids, mask) @ sd["LinearTransformation.weight"].T + sd["LinearTransformation.bias"]
    return out / out.norm(dim=-1, keepdim=True) if normalize else out


@torch.no_grad()
def hf_encode_text(sd, a: dict, ids: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    """The same forward through transformers.XLMRobertaModel / BertModel built from a config (eager attention, no
    dropout) and a torch nn.Linear: what MultilingualCLIP.forward runs, unnormalised."""
    import transformers
    if a["text_kind"] == "xlmr":
        model = transformers.XLMRobertaModel(X.hf_config(_encoder_cfg(a)), add_pooling_layer=False)
    else:
        cfg = transformers.BertConfig(vocab_size=a["vocab"], hidden_size=a["width"], num_hidden_layers=a["layers"],
                                      num_attention_heads=a["heads"], intermediate_size=a["mlp"],
                                      max_position_embeddings=a["max_pos"], type_vocab_size=a["type_vocab"],
                                      pad_token_id=a["pad_id"], layer_norm_eps=a["ln_eps"], hidden_act="gelu",
                                      hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0,
                                      attn_implementation="eager")
        model = transformers.BertModel(cfg, add_pooling_layer=False)
    enc = {k[len(PREFIX):]: v for k, v in sd.items() if k.startswith(PREFIX)}
    missing, unexpected = model.load_state_dict(enc, strict=False)
    assert not unexpected and all("position_ids" in k for k in missing), (missing, unexpected)
    model.eval()
    lin = torch.nn.Linear(a["width"], a["proj_dim"])
    lin.load_state_dict({"weight": sd["LinearTransformation.weight"], "bias": sd["LinearTransformation.bias"]})
    embs = model(input_ids=ids, attention_mask=mask, token_type_ids=torch.zeros_like(ids))[0]
    embs = (embs * mask.unsqueeze(2)).sum(dim=1) / mask.sum(dim=1)[:, None]
    return lin(embs)
