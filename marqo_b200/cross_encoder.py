"""The text reranker's model on the GPU: BERT cross-encoders behind the `CrossEncoder` name Marqo's reranker loads.

A search with `reRanker` set scores its hits with a cross-encoder: `load_sbert_cross_encoder_model`
(reranking/model_utils.py:242-273) builds sentence-transformers' `CrossEncoder(model_name, max_length=512,
device=device, default_activation_function=torch.nn.Sigmoid())`, and `ReRankerText` calls its `predict(pairs)` on the
(query, passage chunk) pairs of the hits (reranking/cross_encoders.py:282-340).  `B200CrossEncoder` has the surface
those two use (`predict`, `tokenizer.model_max_length`, a writable `max_length`) and runs the
BertForSequenceClassification forward in the engine: WordPiece pair encoding with longest_first truncation
(`WordPieceTokenizer`), token types in the BERT embedding, the BERT layers, and the pooler + classifier + sigmoid head
(`Encoder.classify_tokens`).

`register_with_marqo()` replaces the `CrossEncoder` name model_utils looks up with a factory that builds a
`B200CrossEncoder` for the names of `model_registry.CROSS_ENCODER_MODELS` on a CUDA device and the original
sentence-transformers class for every other call.  Marqo keeps everything else: '_testing', 'onnx/...', the model
cache, the sentence split of the hits and the score columns."""
from __future__ import annotations

import json
import os
from typing import Dict, List, Optional, Sequence, Union

import numpy as np

from . import model_registry, weights as weights_mod
from .tokenizers import WordPieceTokenizer

_ACTIVATIONS = {"Sigmoid": True, "Identity": False}   # torch.nn module -> the kernel's sigmoid flag


def _cuda_index(device) -> Optional[int]:
    """The CUDA device index of a torch-style device ("cuda", "cuda:1", 0, torch.device), None for anything else."""
    if isinstance(device, int):
        return device
    s = str(device) if device is not None else ""
    if s == "cuda":
        return 0
    if s.startswith("cuda:") and s[5:].isdigit():
        return int(s[5:])
    return None


def _snapshot_dir(model_name: str) -> str:
    """A local directory holding the model's files: model_name itself, or its snapshot in the Hugging Face cache.
    Nothing is downloaded here; fetching the files stays with the caller."""
    if os.path.isdir(model_name):
        return model_name
    try:
        from huggingface_hub import snapshot_download
        return snapshot_download(repo_id=model_name, local_files_only=True)
    except Exception as e:
        raise OSError(f"{model_name}: no local snapshot (download it into the Hugging Face cache first, or pass "
                      f"`weights` and `vocab_file`): {e}") from e


def _arch_from_config(cfg: dict, model_name: str) -> dict:
    """The engine's BERT block of a BertForSequenceClassification config.json."""
    if cfg.get("model_type") != "bert" or cfg.get("hidden_act", "gelu") != "gelu" or \
            float(cfg.get("layer_norm_eps", 1e-12)) != 1e-12:
        raise ValueError(f"{model_name}: only BERT cross-encoders (erf-GELU, LayerNorm eps 1e-12) are served")
    labels = cfg.get("num_labels") or len(cfg.get("id2label") or {}) or 2
    return {"width": cfg["hidden_size"], "layers": cfg["num_hidden_layers"], "heads": cfg["num_attention_heads"],
            "mlp": cfg["intermediate_size"], "vocab": cfg["vocab_size"],
            "max_pos": cfg.get("max_position_embeddings", 512), "type_vocab": cfg.get("type_vocab_size", 2),
            "num_labels": int(labels)}


class B200CrossEncoder:
    """sentence-transformers 2.2.2 CrossEncoder (verify) for BERT sequence classifiers, on one GPU.

    Weights and vocabulary come from `weights` (a state dict under BertForSequenceClassification's names, or a path
    to one) or `random_init` (a seed, with the registry's shapes) together with `vocab_file`; otherwise from
    model_name's local snapshot directory (config.json, vocab.txt, tokenizer_config.json, model.safetensors or
    pytorch_model.bin)."""

    def __init__(self, model_name: str, max_length: int = 512, device=None, default_activation_function=None,
                 weights=None, random_init: Optional[int] = None, vocab_file=None, max_batch: int = 256):
        index = _cuda_index(device)
        if index is None:
            raise ValueError(f"B200CrossEncoder runs on a CUDA device, not {device!r} (there is no CPU fallback)")
        entry = model_registry.CROSS_ENCODER_MODELS.get(model_name)
        arch = dict(entry["arch"]) if entry else None
        model_max_length, lower = 512, True
        if weights is None and random_init is None:
            root = _snapshot_dir(model_name)
            with open(os.path.join(root, "config.json")) as f:
                arch = _arch_from_config(json.load(f), model_name)
            tc = os.path.join(root, "tokenizer_config.json")
            if os.path.exists(tc):
                with open(tc) as f:
                    t = json.load(f)
                model_max_length = int(min(t.get("model_max_length", 512), 512))
                lower = bool(t.get("do_lower_case", True))
            vocab_file = vocab_file or os.path.join(root, "vocab.txt")
            for fn in ("model.safetensors", "pytorch_model.bin"):
                if os.path.exists(os.path.join(root, fn)):
                    weights = os.path.join(root, fn)
                    break
            else:
                raise OSError(f"{root}: no model.safetensors or pytorch_model.bin")
        if arch is None:
            raise ValueError(f"{model_name} is not a served cross-encoder: its shapes come from a snapshot's config.json")
        if weights is None:
            weights = weights_mod.random_cross_encoder_weights(arch, int(random_init))
        elif isinstance(weights, (str, os.PathLike)):
            weights = weights_mod.load_state_dict(str(weights))
        if vocab_file is None:
            raise ValueError(f"{model_name}: `vocab_file` (vocab.txt) is needed with `weights` / `random_init`")
        from .engine import Encoder
        self.model_name = model_name
        self.num_labels = int(arch["num_labels"])
        self.tokenizer = WordPieceTokenizer(vocab_file, do_lower_case=lower, model_max_length=model_max_length)
        self.max_length = max_length
        self.default_activation_function = default_activation_function
        # BertForSequenceClassification checkpoints also hold the position_ids buffer, which the forward does not read
        sd = {k: v for k, v in weights.items() if not k.endswith("position_ids")}
        self.encoder = Encoder("bert", arch, sd, device=index, max_batch=max_batch)

    def close(self) -> None:
        enc, self.encoder = getattr(self, "encoder", None), None
        if enc is not None:
            enc.close()

    def _sigmoid_flag(self, activation_fct) -> bool:
        if activation_fct is None:
            activation_fct = self.default_activation_function
        if activation_fct is None:   # CrossEncoder's default: Sigmoid for one label, Identity otherwise
            return self.num_labels == 1
        name = type(activation_fct).__name__
        if name not in _ACTIVATIONS or type(activation_fct).__module__.split(".")[0] != "torch":
            raise ValueError(f"activation {activation_fct!r} is not served: torch.nn.Sigmoid() or torch.nn.Identity()")
        return _ACTIVATIONS[name]

    def predict(self, sentences: Sequence, batch_size: int = 32, show_progress_bar=None, num_workers: int = 0,
                activation_fct=None, apply_softmax: bool = False, convert_to_numpy: bool = True,
                convert_to_tensor: bool = False) -> Union[np.ndarray, List, float]:
        """Scores of (text_a, text_b) pairs, as CrossEncoder.predict: each text is strip()-ed, every batch of
        batch_size pairs is tokenised to its own longest row (longest_first truncation at max_length), and the logits
        go through the activation (then a softmax over the labels if apply_softmax and there is more than one).  One
        label gives one score per pair; a single pair (a list of two str) gives one score."""
        if self.encoder is None:
            raise RuntimeError("B200CrossEncoder is closed")
        sigmoid = self._sigmoid_flag(activation_fct)
        single = len(sentences) > 0 and isinstance(sentences[0], str)
        pairs = [sentences] if single else list(sentences)
        for i, p in enumerate(pairs):
            if len(p) != 2:
                raise ValueError(f"pair {i} has {len(p)} texts: a cross-encoder scores (text_a, text_b) pairs")
        scores = np.empty((len(pairs), self.num_labels), np.float32)
        for o in range(0, len(pairs), max(1, int(batch_size))):
            part = pairs[o:o + max(1, int(batch_size))]
            tok = self.tokenizer([str(a).strip() for a, _ in part], [str(b).strip() for _, b in part], padding=True,
                                 truncation="longest_first", max_length=int(self.max_length))
            scores[o:o + len(part)] = self.encoder.classify_tokens(tok["input_ids"], tok["attention_mask"],
                                                                   tok["token_type_ids"], sigmoid=sigmoid)
        if apply_softmax and self.num_labels > 1:
            e = np.exp(scores - scores.max(axis=1, keepdims=True))
            scores = e / e.sum(axis=1, keepdims=True)
        out = scores[:, 0] if self.num_labels == 1 else scores
        if convert_to_tensor:
            import torch
            out = torch.from_numpy(np.ascontiguousarray(out))
        elif not convert_to_numpy:
            import torch
            out = [torch.from_numpy(np.asarray(r)) for r in out]
        return out[0] if single else out


def make_cross_encoder_factory(original, served=B200CrossEncoder):
    """A stand-in for the `CrossEncoder` class: `served` for the names of CROSS_ENCODER_MODELS on a CUDA device,
    `original` (sentence-transformers' class) for every other name or device, with the caller's arguments."""
    def factory(model_name, *args, **kwargs):
        kw = dict(zip(("num_labels", "max_length", "device"), args))   # CrossEncoder's positional order
        kw.update(kwargs)
        if model_name in model_registry.CROSS_ENCODER_MODELS and _cuda_index(kw.get("device")) is not None:
            kw.pop("num_labels", None)   # the checkpoint's own
            return served(model_name, **kw)
        return original(model_name, *args, **kwargs)

    factory.original = original
    return factory


def register_with_marqo() -> None:
    """Serve Marqo's text rerankers on the GPU: replace the CrossEncoder that reranking/model_utils.py calls with the
    factory above (see INTEGRATION.md).  Calling it again keeps the first original."""
    from marqo.s2_inference.reranking import model_utils  # type: ignore
    original = getattr(model_utils.CrossEncoder, "original", model_utils.CrossEncoder)
    model_utils.CrossEncoder = make_cross_encoder_factory(original)
