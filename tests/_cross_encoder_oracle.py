"""ORACLE — TEST INFRASTRUCTURE ONLY.  CPU fp32 restatement of the cross-encoder forward Marqo's text reranker runs:
sentence-transformers 2.2.2 CrossEncoder.predict (verify) over transformers' BertForSequenceClassification (eval mode):

    texts   = [a.strip() for each pair], [b.strip() ...]                # smart_batching_collate_text_only
    tok     = tokenizer(texts_a, texts_b, padding=True, truncation='longest_first', max_length=max_length)
    x       = LN(word[ids] + token_type[type_ids] + position[s])        # BertEmbeddings, eps 1e-12
    x       = BertEncoder(x, key mask from attention_mask)              # post-LN layers, erf-GELU
    pooled  = tanh(pooler.dense(x[:, 0]))                               # BertPooler
    logits  = classifier(pooled)                                        # dropout is a no-op in eval mode
    scores  = Sigmoid(logits)[:, 0]                                     # one label

in batches of batch_size pairs, each padded to its own longest row.  Tested against
transformers.BertForSequenceClassification built from a BertConfig (tests/test_cross_encoder.py)."""
from __future__ import annotations

import copy
import math
from typing import Dict, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

EPS = 1e-12


def arch(name: str, **edits) -> dict:
    """The registry arch of cross-encoder `name` with the given fields changed (layers=2, vocab=1000, ...)."""
    from marqo_b200 import model_registry as R
    a = copy.deepcopy(R.CROSS_ENCODER_MODELS[name]["arch"])
    a.update(edits)
    return a


def weights(a: dict, seed: int) -> Dict[str, torch.Tensor]:
    """The engine's seeded cross-encoder weights (marqo_b200.weights.random_cross_encoder_weights) as torch tensors."""
    from marqo_b200.weights import random_cross_encoder_weights
    return {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in random_cross_encoder_weights(a, seed).items()}


def _long(t) -> torch.Tensor:
    return (t if isinstance(t, torch.Tensor) else torch.as_tensor(np.asarray(t))).long()


@torch.no_grad()
def forward(sd, a: dict, ids, mask, type_ids) -> Tuple[torch.Tensor, torch.Tensor]:
    """(pooled fp32 [n, width], logits fp32 [n, num_labels]) of right-padded pair rows ids, mask, type_ids [n, S]."""
    ids, mask, type_ids = (_long(t) for t in (ids, mask, type_ids))
    B, S = ids.shape
    w, H = a["width"], a["heads"]
    hd = w // H
    p = "bert."
    x = (sd[p + "embeddings.word_embeddings.weight"][ids] + sd[p + "embeddings.token_type_embeddings.weight"][type_ids]
         + sd[p + "embeddings.position_embeddings.weight"][:S])
    x = F.layer_norm(x, (w,), sd[p + "embeddings.LayerNorm.weight"], sd[p + "embeddings.LayerNorm.bias"], EPS)
    add_mask = (1.0 - mask[:, None, None, :].float()) * torch.finfo(torch.float32).min
    for i in range(a["layers"]):
        q_ = f"{p}encoder.layer.{i}."
        lin = lambda t, name: F.linear(t, sd[q_ + name + ".weight"], sd[q_ + name + ".bias"])
        q, k, v = (lin(x, f"attention.self.{nm}").view(B, S, H, hd).transpose(1, 2) for nm in ("query", "key", "value"))
        att = ((q @ k.transpose(-1, -2)) / math.sqrt(hd) + add_mask).softmax(dim=-1)
        o = lin((att @ v).transpose(1, 2).reshape(B, S, w), "attention.output.dense")
        x = F.layer_norm(o + x, (w,), sd[q_ + "attention.output.LayerNorm.weight"],
                         sd[q_ + "attention.output.LayerNorm.bias"], EPS)
        h = lin(F.gelu(lin(x, "intermediate.dense")), "output.dense")
        x = F.layer_norm(h + x, (w,), sd[q_ + "output.LayerNorm.weight"], sd[q_ + "output.LayerNorm.bias"], EPS)
    pooled = torch.tanh(F.linear(x[:, 0], sd[p + "pooler.dense.weight"], sd[p + "pooler.dense.bias"]))
    return pooled, F.linear(pooled, sd["classifier.weight"], sd["classifier.bias"])


def predict(sd, a: dict, tokenizer, pairs: Sequence[Sequence[str]], max_length: int, batch_size: int = 32,
            sigmoid: bool = True) -> np.ndarray:
    """CrossEncoder.predict with one label: fp32 [len(pairs)] scores; `tokenizer` is called as CrossEncoder calls its
    tokenizer (any WordPiece tokenizer with that call)."""
    out = []
    for o in range(0, len(pairs), batch_size):
        part = pairs[o:o + batch_size]
        tok = tokenizer([x.strip() for x, _ in part], [y.strip() for _, y in part], padding=True,
                        truncation="longest_first", max_length=max_length)
        _, logits = forward(sd, a, tok["input_ids"], tok["attention_mask"], tok["token_type_ids"])
        out.append((torch.sigmoid(logits) if sigmoid else logits)[:, 0])
    return torch.cat(out).numpy()


@torch.no_grad()
def hf_forward(sd, a: dict, ids, mask, type_ids) -> Tuple[torch.Tensor, torch.Tensor]:
    """The same through transformers.BertForSequenceClassification built from a BertConfig (eager attention, eval
    mode): (its pooler output, its logits)."""
    import transformers
    cfg = transformers.BertConfig(vocab_size=a["vocab"], hidden_size=a["width"], num_hidden_layers=a["layers"],
                                  num_attention_heads=a["heads"], intermediate_size=a["mlp"],
                                  max_position_embeddings=a["max_pos"], type_vocab_size=a["type_vocab"],
                                  num_labels=a["num_labels"], layer_norm_eps=EPS, hidden_act="gelu",
                                  attn_implementation="eager")
    model = transformers.BertForSequenceClassification(cfg)
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not unexpected and all("position_ids" in k for k in missing), (missing, unexpected)
    model.eval()
    ids, mask, type_ids = (_long(t) for t in (ids, mask, type_ids))
    out = model.bert(input_ids=ids, attention_mask=mask, token_type_ids=type_ids)
    return out.pooler_output, model(input_ids=ids, attention_mask=mask, token_type_ids=type_ids).logits
