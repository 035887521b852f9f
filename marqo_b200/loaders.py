"""Loader classes behind the reference's loader-registry seam (boundary B1, SURVEY §8b).

`MODEL_PROPERTIES['loaders'][type]` (src/marqo/s2_inference/model_registry.py:2133-2145) maps a model `type` to a class
that is constructed as `loader(device=, model_properties=, model_auth=)`, `.load()`-ed once and then driven only
through `.encode(...)` (+ `.preprocess`, `.encode_image`, `.encode_text` on CLIP-type models)
(src/marqo/s2_inference/s2_inference.py:520-568, :129-146, :228-233).  These two classes provide exactly that
surface on top of the C ABI:

  B200OpenCLIP    <-> OPEN_CLIP        (src/marqo/core/inference/embedding_models/open_clip_model.py:249-286,
                                        abstract_clip_model.py:56-112)
  B200HuggingFace <-> HuggingFaceModel (src/marqo/core/inference/embedding_models/hugging_face_model.py:172-214)
  B200HuggingFaceStella <-> HuggingFaceStellaModel (hugging_face_stella_model.py): B200HuggingFace over the GTE
                        runtime, refusing properties without trustRemoteCode
  B200Clip        <-> CLIP             (src/marqo/s2_inference/clip_utils.py:295-492): B200OpenCLIP over OpenAI's
                                        checkpoints, whose arch it reads from a custom checkpoint's shapes
  B200Fp16Clip    <-> FP16_CLIP        (clip_utils.py:495-518): B200Clip returning float16 vectors
  B200MultilingualClip <-> MULTILINGUAL_CLIP (clip_utils.py:521-596): B200Clip's image tower beside M-CLIP's XLM-R or
                                        LaBSE text tower with its projected head

Weights: `model_properties["weights"]` is a state dict (checkpoint names) or a path to one; `"random_init": seed`
builds seeded random weights (benchmarks / self-test).  Tokenisers, in order of preference:
`model_properties["tokenizer"]` (a callable); `model_properties["vocab_file"]` (HF: vocab.txt) /
`model_properties["merges_file"]` (CLIP: bpe_simple_vocab_16e6.txt[.gz]) -> the C++ tokenizers behind the C ABI
(marqo_b200/tokenizers.py, §8 f2); else the HF loader tries `transformers.AutoTokenizer.from_pretrained(name)` and the
CLIP loader `open_clip.get_tokenizer` — both need files that only exist where Marqo's own model cache does.
"""
from __future__ import annotations

import os
from typing import Callable, Dict, List, Optional, Union

import numpy as np

from . import model_registry, weights as weights_mod
from .errors import InternalError, InvalidModelPropertiesError, ModelLoadError, VectoriseError
from .s2_inference import Modality, UnidentifiedImageError, _is_image, _is_tensor, _validate_device


def _resolve_weights(props: dict, arch: dict, kind: str) -> Dict[str, np.ndarray]:
    w = props.get("weights")
    if w is None and props.get("random_init") is not None:
        return weights_mod.random_weights(kind, arch, int(props["random_init"]))
    if w is None:
        raise ModelLoadError("model_properties needs `weights` (state dict or checkpoint path) or `random_init`; "
                             "checkpoint download is Marqo's job (open_clip_model.py:107-131) and out of scope here")
    if isinstance(w, (str, bytes)) or hasattr(w, "__fspath__"):
        w = weights_mod.load_state_dict(w)
    if kind in ("bert", "mpnet", "xlmr"):
        w = weights_mod.strip_hf_prefix(w)
    return w


class _PreprocessToU8:
    """`model.preprocess` replacement (read at s2_inference.py:228-233, applied in the download threads at
    src/marqo/tensor_search/add_docs.py:129-134).  The reference runs Resize+CenterCrop+ToTensor+Normalize on the CPU
    thread; here the thread only hands the decoded pixels over as a uint8 HWC tensor and the whole transform runs on
    the GPU fused into the patch-embed load."""

    def __init__(self, gpu_decode: bool = True):
        self.gpu_decode = gpu_decode

    def __call__(self, pil_image):
        import torch
        if self.gpu_decode:
            # Image.open() is lazy: a JPEG that has not been decoded yet is handed over still encoded and decoded on
            # the GPU with the rest of its batch (image_decode.py, b200_jpeg_decode_batch — bit-exact with Pillow)
            from .image_decode import EncodedImage, encoded_bytes_of
            data = encoded_bytes_of(pil_image)
            if data is not None:
                return EncodedImage(data, "JPEG")
        return torch.from_numpy(np.asarray(pil_image.convert("RGB"), dtype=np.uint8).copy())


class B200OpenCLIP:
    def __init__(self, device: Optional[str] = None, model_properties: Optional[dict] = None, model_auth=None):
        if device is None:
            raise ModelLoadError("`device` is required for loading CLIP models!")  # open_clip_model.py:__init__
        self.device = device
        self.model_properties = dict(model_properties or {})
        self.model_auth = model_auth
        self.model = None
        self.tokenizer: Optional[Callable] = None
        self.preprocess = _PreprocessToU8()
        self.preprocess_config = None

    def load(self) -> None:
        self._load(None)

    def _load(self, state_dict: Optional[Dict[str, np.ndarray]]) -> None:
        """load(), with the weights already read when state_dict is given: the Encoder takes them, and nothing keeps
        the host copy once it is built."""
        from .engine import Encoder
        props = self.model_properties
        arch = props.get("arch")
        if arch is None:
            raise InvalidModelPropertiesError("model_properties has no `arch` block")
        if props.get("mean") is not None:  # open_clip_model_properties.py:24-61 overrides
            arch = dict(arch, mean=tuple(props["mean"]))
        if props.get("std") is not None:
            arch = dict(arch, std=tuple(props["std"]))
        self.arch = arch
        # "siglip" (model_registry.SIGLIP_MODELS): the engine's SigLIP runtime, whose GPU resize squashes images to
        # S x S; "clip_resnet" (RESNET_MODELS): OpenAI's ResNet CLIP; "clip_convnext" (CONVNEXT_MODELS): ConvNeXt
        # CLIP; "clip_eva" (EVA02_MODELS): EVA02 CLIP; otherwise open_clip CLIP; all four shortest side -> S + centre
        # crop (unless the arch asks for the squash)
        kind = arch.get("kind", "clip")
        weights = state_dict if state_dict is not None else _resolve_weights(props, arch, kind)
        self.model = Encoder(kind, arch, weights, device=_validate_device(self.device),
                             max_batch=int(props.get("max_batch", 256)))
        # SigLIP's SentencePiece tokenizer is not restated here: its text needs model_properties["tokenizer"]
        self.tokenizer = props.get("tokenizer") or (None if kind == "siglip" else self._default_tokenizer())

    def _default_tokenizer(self):
        if self.model_properties.get("merges_file"):
            from .tokenizers import ClipBpeTokenizer
            # the CLIP text tower's ctx: in its "text" block, or at the top level of a clip_resnet / clip_convnext /
            # clip_eva arch
            top = self.arch.get("kind") in ("clip_resnet", "clip_convnext", "clip_eva")
            ctx = self.arch["ctx"] if top else self.arch["text"]["ctx"]
            # CoCa's text tower appends its CLS row to ctx - 1 ids (open_clip's CoCa tokenizer context)
            if not top and self.arch["text"].get("embed_cls"):
                ctx -= 1
            return ClipBpeTokenizer(self.model_properties["merges_file"], context_length=int(ctx))
        try:
            import open_clip  # type: ignore
            return open_clip.get_tokenizer(self.model_properties.get("name", "").split("/")[1])
        except Exception:
            return None  # encode_text raises a clear error if text arrives without a tokenizer

    def close(self) -> None:
        if self.model is not None:
            self.model.close()
            self.model = None

    # -- reference surface -------------------------------------------------------------------------------------
    def encode(self, inputs, default: str = 'text', normalize=True, **kwargs) -> np.ndarray:
        """abstract_clip_model.py:56-75"""
        infer = kwargs.pop('infer', True)
        if infer and _is_image(inputs):
            is_image = True
        else:
            if default == 'text':
                is_image = False
            elif default == 'image':
                is_image = True
            else:
                raise UnidentifiedImageError(f"expected default='image' or default='text' but received {default}")
        if is_image:
            return self.encode_image(inputs, normalize=normalize,
                                     image_download_headers=kwargs.get("image_download_headers", dict()))
        return self.encode_text(inputs, normalize=normalize)

    def encode_image(self, images, image_download_headers: Optional[Dict] = None, normalize=True) -> np.ndarray:
        """open_clip_model.py:249-266.  List elements may be PIL images, uint8 HWC tensors/arrays (what
        `self.preprocess` returns) or already-preprocessed float CHW tensors (passed through unchanged by the
        reference, abstract_clip_model.py:108-111)."""
        if self.model is None:
            self.load()
        items = images if isinstance(images, list) else [images]
        if len(items) == 0:
            raise UnidentifiedImageError("received empty list, expected at least one element.")
        S = self.model.image_size
        from .image_decode import EncodedImage, decode_images_to_device
        if any(isinstance(it, (EncodedImage, bytes, bytearray)) for it in items):
            # still-encoded files (what the preprocessor hands over for JPEGs): decode the batch on the GPU; the pixels
            # stay in HBM for the resize + patch-embed kernels
            enc_idx = [i for i, it in enumerate(items) if isinstance(it, (EncodedImage, bytes, bytearray))]
            try:
                decoded = decode_images_to_device([items[i] for i in enc_idx], device=self.model.device)
            except OSError as e:              # Pillow's error for broken files, wrapped like the reference does
                raise UnidentifiedImageError(str(e)) from e
            items = list(items)
            for i, t in zip(enc_idx, decoded):
                items[i] = t
        if all(self._on_model_device(it) for it in items):
            return self._encode_device_images(items, bool(normalize))
        u8, f32 = [], []
        for it in items:
            if isinstance(it, str):
                raise VectoriseError("image download is Marqo's job (image_download.py:130-215); pass decoded images")
            if type(it).__module__.startswith("PIL."):
                it = np.asarray(it.convert("RGB"), dtype=np.uint8)
            if _is_tensor(it):
                it = it.detach().to("cpu").numpy()
            a = np.asarray(it)
            if a.dtype == np.uint8 and a.ndim == 3 and a.shape[2] == 3:
                u8.append(a)
            elif a.dtype.kind == "f" and a.shape == (3, S, S):
                f32.append(a.astype(np.float32, copy=False))
            else:
                raise UnidentifiedImageError(f"unsupported image element: dtype {a.dtype}, shape {a.shape}")
        if u8 and f32:
            raise UnidentifiedImageError("a batch must not mix raw uint8 images and preprocessed tensors")
        if f32:
            return self.model.encode_images_f32(np.stack(f32), normalize=bool(normalize))
        out = np.empty((len(u8), self.model.embed_dim), np.float32)
        # group by (h, w): the C ABI takes one rectangular uint8 block per call
        groups: Dict[tuple, List[int]] = {}
        for i, a in enumerate(u8):
            groups.setdefault(a.shape[:2], []).append(i)
        for (h, w), idx in groups.items():
            out[idx] = self.model.encode_images_u8_list([u8[i] for i in idx], normalize=bool(normalize))
        return out

    def _on_model_device(self, it) -> bool:
        """A uint8 HWC torch tensor already resident on this model's GPU — what Marqo's download threads produce:
        `preprocessors['image'](image).to(device)` (add_docs.py:129-134)."""
        return (_is_tensor(it) and getattr(it, "is_cuda", False) and it.device.index == self.model.device
                and str(it.dtype) == "torch.uint8" and it.ndim == 3 and it.shape[2] == 3)

    def _encode_device_images(self, items, normalize: bool) -> np.ndarray:
        """Images that are already in HBM stay there: one device-side stack per image size, the device entry point,
        one D2H copy of the [n, dim] result — no per-image round trip through the host."""
        import torch
        out = torch.empty((len(items), self.model.embed_dim), dtype=torch.float32, device=items[0].device)
        groups: Dict[tuple, List[int]] = {}
        for i, t in enumerate(items):
            groups.setdefault((int(t.shape[0]), int(t.shape[1])), []).append(i)
        for (h, w), idx in groups.items():
            batch = torch.stack([items[i] for i in idx]).contiguous()
            res = out if len(groups) == 1 else torch.empty((len(idx), self.model.embed_dim), dtype=torch.float32,
                                                          device=batch.device)
            self._sync_device(batch.device)      # the engine runs on its own stream: the stack must have landed
            self.model.encode_images_u8_device(batch.data_ptr(), len(idx), h, w, res.data_ptr(), normalize=normalize,
                                               sync=True)
            if res is not out:
                out[torch.as_tensor(idx, device=out.device)] = res
        return out.cpu().numpy()

    @staticmethod
    def _sync_device(device) -> None:
        import torch
        torch.cuda.synchronize(device)

    def _tokenize(self, sentence) -> np.ndarray:
        if self.tokenizer is None:
            if self.arch.get("kind") == "siglip":
                raise ModelLoadError("no SigLIP tokenizer available: supply model_properties['tokenizer'], a callable "
                                     "returning [n, 64] token ids (SigLIP's SentencePiece vocabulary is not bundled)")
            raise ModelLoadError("no CLIP tokenizer available: supply model_properties['tokenizer'] "
                                 "(open_clip's BPE vocabulary is not bundled)")
        text = self.tokenizer(sentence if isinstance(sentence, list) else [sentence])
        if _is_tensor(text):
            text = text.detach().to("cpu").numpy()
        return np.ascontiguousarray(text, dtype=np.int32)

    def encode_text(self, sentence: Union[str, List[str]], normalize=True) -> np.ndarray:
        """open_clip_model.py:268-286"""
        if self.model is None:
            self.load()
        return self.model.encode_tokens(self._tokenize(sentence), None, normalize=bool(normalize))

    # -- add_documents fast path: embeddings stay in HBM (consumed by GpuTensorIndex.feed_batch as DeviceChunks) ----
    def encode_to_device(self, inputs, default: str = 'text', normalize=True, sub_batch: int = 256, **kwargs):
        """encode() whose result is a CUDA fp32 tensor [n, dim] on the model's device instead of a host ndarray: the
        vectors go from the projection + L2 epilogue straight into the row store (b200_index_add_device_docs), never
        through `List[List[float]]`.  Same routing rules as encode() (abstract_clip_model.py:56-75).  Images: uint8 HWC
        arrays / tensors; a sub-batch of one size is stacked into one block, one of mixed sizes goes to the ragged entry
        point in one call (CUDA tensors by pointer, host arrays in one packed upload).  Texts: strings, or an int32
        [n, ctx] array of token ids."""
        import torch
        if self.model is None:
            self.load()
        infer = kwargs.pop('infer', True)
        items = inputs if isinstance(inputs, list) else [inputs]
        is_ids = isinstance(inputs, np.ndarray) and inputs.dtype.kind in "iu" and inputs.ndim == 2
        is_image = not is_ids and ((infer and _is_image(inputs)) or default == 'image')
        dev = self._torch_device()
        n = inputs.shape[0] if is_ids else len(items)
        out = torch.empty((n, self.model.embed_dim), dtype=torch.float32, device=dev)
        step = max(1, min(int(sub_batch), int(self.model_properties.get("max_batch", 256))))
        if is_image:
            for lo in range(0, n, step):
                part = items[lo:lo + step]
                on_device = all(self._on_model_device(it) for it in part)
                if not on_device:
                    part = [np.asarray(it.cpu() if _is_tensor(it) else
                                       (it.convert("RGB") if type(it).__module__.startswith("PIL.") else it),
                                       dtype=np.uint8) for it in part]
                if len({tuple(it.shape) for it in part}) > 1:
                    self._encode_ragged_to_device(part, on_device, out[lo:], bool(normalize))
                    continue
                if on_device:
                    batch = torch.stack(part).contiguous()
                else:
                    batch = torch.from_numpy(np.stack(part)).to(dev, non_blocking=False)
                if batch.ndim != 4 or batch.shape[3] != 3:
                    raise UnidentifiedImageError(f"expected uint8 [n, H, W, 3] images, got {tuple(batch.shape)}")
                self._sync_device(dev)
                self.model.encode_images_u8_device(batch.data_ptr(), len(part), int(batch.shape[1]), int(batch.shape[2]),
                                                   out[lo:].data_ptr(), normalize=bool(normalize), sync=True)
        else:
            ids = np.ascontiguousarray(inputs, dtype=np.int32) if is_ids else self._tokenize(items)
            d_ids = torch.from_numpy(ids).to(dev)
            self._sync_device(dev)
            for lo in range(0, n, step):
                m = min(step, n - lo)
                self.model.encode_tokens_device(d_ids[lo:].data_ptr(), None, m, int(ids.shape[1]), out[lo:].data_ptr(),
                                                normalize=bool(normalize), sync=True)
        return out

    def _encode_ragged_to_device(self, part, on_device: bool, out, normalize: bool) -> None:
        """Images of mixed sizes (CUDA tensors on the model's device, or host arrays) -> rows out[:len(part)] through
        one ragged call; host arrays are packed back to back and uploaded in one copy."""
        import torch
        for it in part:
            if it.ndim != 3 or it.shape[2] != 3:
                raise UnidentifiedImageError(f"expected uint8 [H, W, 3] images, got {tuple(it.shape)}")
        if on_device:
            keep = [t.contiguous() for t in part]
            ptrs = [t.data_ptr() for t in keep]
        else:
            keep = torch.from_numpy(np.concatenate([a.reshape(-1) for a in part])).to(self._torch_device(),
                                                                                      non_blocking=False)
            offsets = np.cumsum([0] + [a.size for a in part[:-1]])
            ptrs = [keep.data_ptr() + int(o) for o in offsets]
        self._sync_device(out.device)
        self.model.encode_images_u8_ragged_device(ptrs, [int(it.shape[0]) for it in part],
                                                  [int(it.shape[1]) for it in part], out.data_ptr(),
                                                  normalize=normalize, sync=True)

    def _torch_device(self):
        """The torch device of the model's GPU, where encode_to_device's results live."""
        import torch
        return torch.device("cuda", self.model.device)


class B200HuggingFace:
    def __init__(self, device: Optional[str] = None, model_properties: Optional[dict] = None, model_auth=None):
        if device is None:
            raise ModelLoadError("`device` is required for loading HF models!")
        self.device = device
        self.model_properties = dict(model_properties or {})
        self.model_auth = model_auth
        self._model = None
        self._tokenizer = None
        self.max_seq_length = int(self.model_properties.get("tokens", 128))

    def load(self) -> None:
        from .engine import Encoder
        props = self.model_properties
        arch = props.get("arch")
        if arch is None:
            raise InvalidModelPropertiesError("model_properties has no `arch` block")
        if props.get("poolingMethod") or props.get("pooling_method"):  # hugging_face_model_properties.py
            arch = dict(arch, pool=(props.get("poolingMethod") or props.get("pooling_method")))
        self.arch = arch
        # "mpnet": MPNetModel (model_registry.MPNET_MODELS); "xlmr": XLMRobertaModel (XLMR_MODELS); "gte": NewModel
        # (GTE_MODELS); else BertModel
        kind = arch.get("kind", "bert")
        self._model = Encoder(kind, arch, _resolve_weights(props, arch, kind), device=_validate_device(self.device),
                              max_batch=int(props.get("max_batch", 256)))
        self._tokenizer = props.get("tokenizer") or self._default_tokenizer()

    def _default_tokenizer(self):
        vocab_file = self.model_properties.get("vocab_file")
        if vocab_file:
            from .tokenizers import MPNetTokenizer, WordPieceTokenizer, XLMRTokenizer, is_sentencepiece_model
            if is_sentencepiece_model(vocab_file):   # sentencepiece.bpe.model (multilingual-e5)
                return XLMRTokenizer(vocab_file)
            cls = MPNetTokenizer if self.arch.get("kind") == "mpnet" else WordPieceTokenizer
            return cls(self.model_properties["vocab_file"],
                       do_lower_case=bool(self.model_properties.get("do_lower_case", True)))
        try:
            from transformers import AutoTokenizer
            return AutoTokenizer.from_pretrained(self.model_properties["name"])
        except Exception:
            return None

    def close(self) -> None:
        if self._model is not None:
            self._model.close()
            self._model = None

    def encode(self, sentence: Union[str, List[str]], normalize=True, **kwargs) -> np.ndarray:
        """hugging_face_model.py:172-197: tokenizer(padding=True, truncation=True, max_length=tokens) -> forward ->
        pooling -> F.normalize."""
        if isinstance(sentence, str):
            sentence = [sentence]
        if self._model is None:
            self.load()
        if self._tokenizer is None:
            raise ModelLoadError("no tokenizer available: supply model_properties['tokenizer'] or make "
                                 f"{self.model_properties.get('name')!r} loadable by transformers.AutoTokenizer")
        tok = self._tokenizer(sentence, padding=True, truncation=True, max_length=self.max_seq_length,
                              return_tensors="np")
        ids = np.asarray(tok["input_ids"], dtype=np.int32)
        mask = np.asarray(tok["attention_mask"], dtype=np.int32)
        return self._model.encode_tokens(ids, mask, normalize=bool(normalize))

    def encode_to_device(self, sentence, normalize=True, sub_batch: int = 64, attention_mask=None, **kwargs):
        """encode() whose result stays on the GPU (CUDA fp32 tensor [n, dim]) for the add_documents fast path.
        `sentence`: strings (tokenised per sub-batch with padding=True, like the reference's own sub-batching,
        s2_inference.py:137-146), or an int32 [n, seq] array of token ids (+ optional attention_mask)."""
        import torch
        if self._model is None:
            self.load()
        dev = torch.device("cuda", self._model.device)
        is_ids = isinstance(sentence, np.ndarray) and sentence.dtype.kind in "iu" and sentence.ndim == 2
        items = sentence if is_ids else ([sentence] if isinstance(sentence, str) else list(sentence))
        n = len(items)
        out = torch.empty((n, self._model.embed_dim), dtype=torch.float32, device=dev)
        step = max(1, min(int(sub_batch), int(self.model_properties.get("max_batch", 256))))
        for lo in range(0, n, step):
            if is_ids:
                ids = np.ascontiguousarray(items[lo:lo + step], dtype=np.int32)
                mask = None if attention_mask is None else np.ascontiguousarray(attention_mask[lo:lo + step], dtype=np.int32)
            else:
                if self._tokenizer is None:
                    raise ModelLoadError("no tokenizer available: supply model_properties['tokenizer'] or 'vocab_file'")
                tok = self._tokenizer(items[lo:lo + step], padding=True, truncation=True, max_length=self.max_seq_length,
                                      return_tensors="np")
                ids = np.asarray(tok["input_ids"], dtype=np.int32)
                mask = np.asarray(tok["attention_mask"], dtype=np.int32)
            d_ids = torch.from_numpy(ids).to(dev)
            d_mask = None if mask is None else torch.from_numpy(mask).to(dev)
            torch.cuda.synchronize(dev)
            self._model.encode_tokens_device(d_ids.data_ptr(), None if d_mask is None else d_mask.data_ptr(), ids.shape[0],
                                             ids.shape[1], out[lo:].data_ptr(), normalize=bool(normalize), sync=True)
        return out


class B200HuggingFaceStella(B200HuggingFace):
    """The Stella embedder's loader type (model_registry.GTE_MODELS).  The reference loads its checkpoint with
    trust_remote_code and refuses model properties without `trustRemoteCode: True` when the loader is constructed
    (hugging_face_model.py:54-59); so does this one, before any GPU work."""

    def __init__(self, device: Optional[str] = None, model_properties: Optional[dict] = None, model_auth=None):
        if not (model_properties or {}).get("trustRemoteCode"):
            raise InvalidModelPropertiesError(
                "The specified model requires the 'trustRemoteCode' attribute to be set to True. Setting this "
                "attribute to True may have security implications.")
        super().__init__(device=device, model_properties=model_properties, model_auth=model_auth)


WIDE_RESNET_MAX_BATCH = 64   # B200Clip's default max_batch for ResNets wider than 64 (RN50x4, RN50x16, RN50x64)


class B200Clip(B200OpenCLIP):
    """The reference's `clip` loader type (model_registry.OPENAI_CLIP_MODELS: "ViT-B/32", "RN50", ...).  The networks
    are the open_clip */openai ones, run by the same encoders; what differs is the loader's own behaviour:
      - construction without a device raises InternalError, not ModelLoadError (clip_utils.py:305-306);
      - a custom model names its checkpoint by `localpath` (or the engine's own `weights`); `url` and
        `model_location` are refused with ModelLoadError, as downloading is Marqo's job, and more than one of the three
        with InvalidModelPropertiesError (clip_utils.py:360-364);
      - without an `arch` block the arch is read from the checkpoint's shapes (model_registry.openai_clip_arch), as
        clip.load builds the model from its state dict, so any OpenAI-format checkpoint (RN50x4 too) is served;
      - the tokenizer is clip.tokenize(truncate=True): the CLIP BPE at context 77 with EOT forced into the last slot,
        from `merges_file`, else the `clip` package's own when it is importable."""

    def __init__(self, device: Optional[str] = None, model_properties: Optional[dict] = None, model_auth=None):
        if not device:
            raise InternalError("`device` is required for loading CLIP models!")
        super().__init__(device=device, model_properties=model_properties, model_auth=model_auth)

    def load(self) -> None:
        props = self.model_properties
        given = [k for k in ("localpath", "url", "model_location") if props.get(k)]
        if len(given) > 1:
            raise InvalidModelPropertiesError(
                "Only one of `url`, `localpath` or `model_location` can be specified in model_properties. Please "
                "ensure that only one of these is specified in model_properties and retry.")
        if given and given[0] != "localpath":
            raise ModelLoadError(f"model_properties[{given[0]!r}]: downloading the checkpoint is Marqo's job; pass "
                                 "the downloaded file as `localpath`")
        if given:
            path = props["localpath"]
            if not os.path.isfile(path):
                raise InvalidModelPropertiesError(f"Marqo can not load the custom clip model. The provided model path "
                                                  f"`{path}` is not a local file.")
            props = dict(props, weights=path)
        sd = None   # the checkpoint, when it has to be read for its arch; handed to the Encoder, never stored
        if props.get("arch") is None and props.get("weights") is not None:
            sd = props["weights"]
            if isinstance(sd, (str, bytes)) or hasattr(sd, "__fspath__"):
                sd = weights_mod.load_state_dict(sd)
            arch = model_registry.openai_clip_arch(sd)
            if props.get("dimensions") is not None and int(props["dimensions"]) != arch["embed_dim"]:
                raise InvalidModelPropertiesError(
                    f"model_properties declares dimensions {props['dimensions']}, but the checkpoint's "
                    f"text_projection gives embeddings of {arch['embed_dim']}")
            props = dict(props, arch=arch)
        r = (props.get("arch") or {}).get("resnet")
        if r is not None and r["width"] > 64 and props.get("max_batch") is None:
            # the wide ResNets' four activation buffers hold max_batch x (S/2)^2 x width bf16 values each: 7.1 MB
            # (RN50x16) and 12.8 MB (RN50x64) per image, 7.2 and 13 GB at the usual 256 images; at 64 images the
            # models hold 2.2 and 4.2 GB of device memory in all and every trunk GEMM still has >= 9216 rows
            # (DESIGN.md §6)
            props = dict(props, max_batch=WIDE_RESNET_MAX_BATCH)
        self.model_properties = props
        self._load(sd)

    def _default_tokenizer(self):
        if self.model_properties.get("merges_file"):
            return super()._default_tokenizer()
        try:
            import clip  # type: ignore
        except Exception:
            return None  # encode_text raises a clear error if text arrives without a tokenizer
        return lambda texts: clip.tokenize(texts, truncate=True)


class B200Fp16Clip(B200Clip):
    """The reference's `fp16_clip` loader type ("fp16/ViT-B/32", ...).  On CUDA the reference runs the model in fp16
    and returns float16 arrays (clip_utils.py:393-397, 512-518); this loader runs the same encoder as the fp32 name and
    returns its vectors rounded to float16 (encode_to_device: the rounded values, as fp32 for the row store).
    `fp16_clip` is not a preprocess-image type (constants.py:31), so Marqo hands its images over undecoded."""

    def encode_image(self, images, image_download_headers: Optional[Dict] = None, normalize=True) -> np.ndarray:
        return super().encode_image(images, image_download_headers=image_download_headers,
                                    normalize=normalize).astype(np.float16)

    def encode_text(self, sentence: Union[str, List[str]], normalize=True) -> np.ndarray:
        return super().encode_text(sentence, normalize=normalize).astype(np.float16)

    def encode_to_device(self, inputs, default: str = 'text', normalize=True, sub_batch: int = 256, **kwargs):
        out = super().encode_to_device(inputs, default=default, normalize=normalize, sub_batch=sub_batch, **kwargs)
        return out.half().float()


class B200MultilingualClip(B200OpenCLIP):
    """The reference's `multilingual_clip` loader type (model_registry.MULTILINGUAL_CLIP_MODELS).  Two Encoders:
      - the image tower, exactly the one B200Clip builds for the entry's `visual` name (clip.load's visual(x));
      - the text tower, M-CLIP's XLM-R or BERT encoder with its masked-mean LinearTransformation head, run over
        tokenizer(texts, padding=True): the batch padded to its longest text.
    Weights: `visual_weights`, an OpenAI-format CLIP checkpoint of which only visual.* is read, and `textual_weights`,
    the MultilingualCLIP checkpoint (state dicts or paths); `random_init` seeds both instead, the image tower as B200Clip
    seeds it.  Tokenizer: model_properties["tokenizer"] (a callable), else `vocab_file` (XLM-R: sentencepiece.bpe.model
    -> XLMRTokenizer; LaBSE: vocab.txt -> the cased WordPieceTokenizer), else transformers.AutoTokenizer of the
    entry's textual_model.  The reference's tokenizer call does not truncate, so a text longer than the encoder's 512
    positions fails there inside the embedding (torch's IndexError for XLM-R, a size mismatch for LaBSE); here it is
    refused with VectoriseError before any GPU work, never truncated."""

    def __init__(self, device: Optional[str] = None, model_properties: Optional[dict] = None, model_auth=None):
        if not device:
            raise InternalError("`device` is required for loading MULTILINGUAL CLIP models!")
        super().__init__(device=device, model_properties=model_properties, model_auth=model_auth)
        self.text_model = None

    def load(self) -> None:
        from .engine import Encoder
        props = self.model_properties
        arch = props.get("arch")
        if arch is None:
            raise InvalidModelPropertiesError("model_properties has no `arch` block")
        seed = props.get("random_init")
        for k in ("visual_weights", "textual_weights"):
            if props.get(k) is None and seed is None:
                raise ModelLoadError(f"model_properties needs `{k}` (state dict or checkpoint path) or `random_init`; "
                                     "checkpoint download is Marqo's job")
        # B200Clip's image tower: the OPENAI_CLIP_MODELS arch without its text tower
        self.arch = dict(model_registry.OPENAI_CLIP_MODELS[arch["visual"]]["arch"], text=None)
        device, max_batch = _validate_device(self.device), int(props.get("max_batch", 256))
        vis = props.get("visual_weights")
        if vis is None:
            vis = weights_mod.random_clip_weights(self.arch, int(seed))
        elif isinstance(vis, (str, bytes)) or hasattr(vis, "__fspath__"):
            vis = weights_mod.load_state_dict(vis)
        txt = props.get("textual_weights")
        if txt is None:
            txt = weights_mod.random_mclip_text_weights(arch, int(seed) + 1)
        elif isinstance(txt, (str, bytes)) or hasattr(txt, "__fspath__"):
            txt = weights_mod.load_state_dict(txt)
        self.model = Encoder("clip", self.arch, {k: v for k, v in vis.items() if k.startswith("visual.")},
                             device=device, max_batch=max_batch)
        try:
            self.text_model = Encoder(arch["text_kind"], arch, txt, device=device, max_batch=max_batch)
        except Exception:
            self.close()
            raise
        # the encoder's positions: XLM-R's start after the pad id
        self.max_tokens = arch["max_pos"] - (arch["pad_id"] + 1 if arch["text_kind"] == "xlmr" else 0)
        self.tokenizer = props.get("tokenizer") or self._default_tokenizer()

    def _default_tokenizer(self):
        props, kind = self.model_properties, self.model_properties["arch"]["text_kind"]
        if props.get("vocab_file"):
            from .tokenizers import WordPieceTokenizer, XLMRTokenizer
            if kind == "xlmr":
                return XLMRTokenizer(props["vocab_file"])
            return WordPieceTokenizer(props["vocab_file"], do_lower_case=False)
        try:
            from transformers import AutoTokenizer
            return AutoTokenizer.from_pretrained(props["textual_model"])
        except Exception:
            return None  # encode_text raises a clear error if text arrives without a tokenizer

    def close(self) -> None:
        super().close()
        if self.text_model is not None:
            self.text_model.close()
            self.text_model = None

    def _tokens(self, sentences: List[str]):
        """ids and mask int32 [n, L], L the longest text's tokens; a text over max_tokens is refused."""
        if self.tokenizer is None:
            raise ModelLoadError("no M-CLIP tokenizer available: supply model_properties['tokenizer'] or 'vocab_file'")
        # one token past the limit shows a text that does not fit without tokenizing all of a long one
        tok = self.tokenizer(sentences, padding=True, truncation=True, max_length=self.max_tokens + 1,
                             return_tensors="np")
        ids = np.ascontiguousarray(tok["input_ids"], dtype=np.int32)
        mask = np.ascontiguousarray(tok["attention_mask"], dtype=np.int32)
        lens = mask.sum(axis=1)
        if lens.max() > self.max_tokens:
            i = int(np.argmax(lens > self.max_tokens))
            raise VectoriseError(f"text {i} is longer than the {self.max_tokens} tokens the multilingual_clip text "
                                 f"encoder takes; it is not truncated, as the reference's M-CLIP tokenizer call does not "
                                 f"truncate either")
        return ids, mask

    def encode_text(self, sentence: Union[str, List[str]], normalize=True) -> np.ndarray:
        """clip_utils.py:555-570: MultilingualCLIP.forward, then / |out| when normalize is set"""
        if self.text_model is None:
            self.load()
        ids, mask = self._tokens(sentence if isinstance(sentence, list) else [sentence])
        return self.text_model.encode_tokens(ids, mask, normalize=bool(normalize))

    def encode_to_device(self, inputs, default: str = 'text', normalize=True, sub_batch: int = 256, **kwargs):
        """B200OpenCLIP.encode_to_device for images; texts (strings, tokenized per sub-batch) run the text Encoder."""
        import torch
        infer = kwargs.get('infer', True)
        is_ids = isinstance(inputs, np.ndarray) and inputs.dtype.kind in "iu" and inputs.ndim == 2
        if is_ids or (infer and _is_image(inputs)) or default == 'image':
            if is_ids:
                raise VectoriseError("multilingual_clip takes texts as strings: token ids carry no attention mask")
            return super().encode_to_device(inputs, default=default, normalize=normalize, sub_batch=sub_batch, **kwargs)
        if self.text_model is None:
            self.load()
        items = inputs if isinstance(inputs, list) else [inputs]
        dev = self._torch_device()
        out = torch.empty((len(items), self.text_model.embed_dim), dtype=torch.float32, device=dev)
        step = max(1, min(int(sub_batch), int(self.model_properties.get("max_batch", 256))))
        for lo in range(0, len(items), step):
            ids, mask = self._tokens(items[lo:lo + step])
            d_ids, d_mask = torch.from_numpy(ids).to(dev), torch.from_numpy(mask).to(dev)
            self._sync_device(dev)
            self.text_model.encode_tokens_device(d_ids.data_ptr(), d_mask.data_ptr(), ids.shape[0], ids.shape[1],
                                                 out[lo:].data_ptr(), normalize=bool(normalize), sync=True)
        return out


def _read_video_frames(path: str, num_frames: int) -> np.ndarray:
    """LanguageBind's opencv decode (languagebind/video/processing_video.py:80-93): frame ids np.linspace(0, count - 1,
    num_frames, dtype=int) of CAP_PROP_FRAME_COUNT, each read after seeking to it and turned BGR -> RGB.  uint8
    [num_frames, H, W, 3]."""
    import cv2
    cap = cv2.VideoCapture(str(path))
    try:
        count = int(cap.get(cv2.CAP_PROP_FRAME_COUNT))
        frames = []
        for idx in np.linspace(0, count - 1, num_frames, dtype=int):
            cap.set(cv2.CAP_PROP_POS_FRAMES, int(idx))
            ok, frame = cap.read()
            if not ok or frame is None:
                raise VectoriseError(f"Could not read frame {int(idx)} of video {path}")
            frames.append(cv2.cvtColor(frame, cv2.COLOR_BGR2RGB))
    finally:
        cap.release()
    return np.stack(frames)


class LanguageBindVideoPreprocessor:
    """What LanguageBindVideoProcessor(config)(paths) does on the host (processing_video.py:48-99): decode and sample
    the frames of each video file.  Returns {"pixel_values": uint8 [n, T, H, W, 3]} for videos of one size; the
    transform (ShortSideScale, CenterCropVideo, Normalize) runs on the GPU in B200LanguageBind.encode."""

    def __init__(self, num_frames: int):
        self.num_frames = int(num_frames)

    def __call__(self, images=None, return_tensors=None, **kwargs):
        paths = images if isinstance(images, (list, tuple)) else [images]
        videos = [_read_video_frames(p, self.num_frames) for p in paths]
        if len({v.shape for v in videos}) != 1:
            raise VectoriseError("videos of different sizes: preprocess them one at a time")
        return {"pixel_values": np.stack(videos)}


class B200LanguageBind:
    """Marqo's `languagebind` loader (multimodal_model_load.py:204-299, LanguageBindEncoder) for
    LanguageBind/Video_V1.5_FT on the engine: the video tower (LanguageBindVideo.vision_model with its temporal layers,
    video_frames in the arch) and the checkpoint's CLIP text tower in one Encoder.

    Weights: model_properties["weights"] (a LanguageBindVideo state dict or checkpoint file), or `localpath`, a snapshot
    directory with config.json and pytorch_model.bin / model.safetensors, or `random_init` (a seed).  config.json, when
    there is one, gives num_frames, hidden_act, layer_norm_eps and the embedding form (clip_type "vl" or "vl_new", whose
    tube_size must be 1), each checked against the arch; the tensors' shapes are checked by the engine.  Nothing is
    downloaded.  Text is tokenised by model_properties["tokenizer"] or the CLIP BPE of `merges_file` at context 77.

    Outputs follow LanguageBind.forward and the encoder's _normalize: every vector is v / |v|; a video vector is then
    multiplied by exp(logit_scale); normalize=True divides by the norm once more.  Unlike the reference, the video
    transform does not apply RandomHorizontalFlipVideo(p=0.5), which the reference runs at inference and which makes
    its video embeddings random; the engine's are those of the unflipped frames."""

    def __init__(self, device: Optional[str] = None, model_properties: Optional[dict] = None, model_auth=None):
        if device is None:
            raise ModelLoadError("`device` is required for loading LanguageBind models!")
        self.device = device
        self.model_properties = dict(model_properties or {})
        self.model = None
        self.tokenizer: Optional[Callable] = None
        self._preprocessors: Dict[Modality, Callable] = {}

    @staticmethod
    def _check_config(cfg: dict, arch: dict) -> dict:
        """The arch with the act of the checkpoint's config.json (both towers must agree), after checking the fields
        the engine fixes: 8 frames as the arch says, eps 1e-5, a tube of one frame."""
        v, t = cfg.get("vision_config", {}), cfg.get("text_config", {})
        acts = {v.get("hidden_act", "quick_gelu"), t.get("hidden_act", "quick_gelu")}
        if len(acts) != 1 or not acts <= {"gelu", "quick_gelu"}:
            raise InvalidModelPropertiesError(f"LanguageBind: hidden_act {sorted(acts)} is not one gelu / quick_gelu")
        frames = int(v.get("num_frames", 1))
        if frames != arch["video_frames"]:
            raise InvalidModelPropertiesError(f"LanguageBind: num_frames {frames} != the arch's {arch['video_frames']}")
        for c in (v, t):
            if float(c.get("layer_norm_eps", 1e-5)) != 1e-5:
                raise InvalidModelPropertiesError("LanguageBind: the engine's CLIP towers take layer_norm_eps 1e-5")
        if v.get("clip_type", "vl") == "vl_new" and int(v.get("tube_size", 1)) != 1:
            raise InvalidModelPropertiesError("LanguageBind: a patch embedding over tubes of more than one frame")
        return dict(arch, act="gelu" if acts == {"gelu"} else "quickgelu")

    def load(self) -> None:
        import json
        from .engine import Encoder
        props = self.model_properties
        arch = props.get("arch")
        if arch is None or not arch.get("video_frames"):
            raise InvalidModelPropertiesError("model_properties has no LanguageBind `arch` block (video_frames)")
        w = props.get("weights")
        local = props.get("localpath")
        if local and os.path.isdir(local):
            cfg_path = os.path.join(local, "config.json")
            if os.path.exists(cfg_path):
                with open(cfg_path) as f:
                    arch = self._check_config(json.load(f), arch)
            if w is None:
                for fn in ("model.safetensors", "pytorch_model.bin"):
                    if os.path.exists(os.path.join(local, fn)):
                        w = os.path.join(local, fn)
                        break
        if w is None and props.get("random_init") is not None:
            w = weights_mod.random_languagebind_video_weights(arch, int(props["random_init"]))
        if w is None:
            raise ModelLoadError("model_properties needs `weights`, a `localpath` snapshot or `random_init`; "
                                 "checkpoint download is Marqo's job and out of scope here")
        if isinstance(w, (str, bytes)) or hasattr(w, "__fspath__"):
            w = weights_mod.load_state_dict(w)
        self.arch = arch
        self.model = Encoder("clip", arch, weights_mod.languagebind_video_state_dict_to_engine(w),
                             device=_validate_device(self.device), max_batch=int(props.get("max_batch", 32)))
        self.tokenizer = props.get("tokenizer")
        if self.tokenizer is None and props.get("merges_file"):
            from .tokenizers import ClipBpeTokenizer
            self.tokenizer = ClipBpeTokenizer(props["merges_file"], context_length=int(arch["text"]["ctx"]))

    def close(self) -> None:
        if self.model is not None:
            self.model.close()
            self.model = None

    def preprocessor(self, modality):
        """The host preprocessor of a modality this model has (video), else None, as LanguageBindEncoder.preprocessor
        returns for a modality outside its clip_type."""
        if Modality(modality) != Modality.VIDEO:
            return None
        if Modality.VIDEO not in self._preprocessors:
            self._preprocessors[Modality.VIDEO] = LanguageBindVideoPreprocessor(self.arch["video_frames"])
        return self._preprocessors[Modality.VIDEO]

    def _encode_videos(self, videos: List[np.ndarray], normalize: bool) -> np.ndarray:
        """uint8 [T, H, W, 3] videos, grouped by size into one engine call each, rows returned in the input order."""
        out = np.empty((len(videos), self.model.embed_dim), np.float32)
        groups: Dict[tuple, List[int]] = {}
        for i, v in enumerate(videos):
            groups.setdefault(v.shape, []).append(i)
        for idx in groups.values():
            out[idx] = self.model.encode_videos_u8(np.stack([videos[i] for i in idx]), normalize=normalize)
        return out

    def encode(self, content, modality=Modality.TEXT, normalize=True, **kwargs) -> np.ndarray:
        modality = Modality(modality) if modality is not None else Modality.TEXT
        if modality == Modality.TEXT:
            if self.tokenizer is None:
                raise VectoriseError("LanguageBind text needs model_properties['tokenizer'] or a merges_file")
            texts = [content] if isinstance(content, str) else list(content)
            ids = np.asarray(self.tokenizer(texts), dtype=np.int32)
            return self.model.encode_tokens(ids, normalize=normalize)
        if modality == Modality.VIDEO:
            items = [content] if isinstance(content, (str, dict)) or hasattr(content, "__fspath__") else list(content)
            videos: List[np.ndarray] = []
            for it in items:
                if isinstance(it, dict) and "pixel_values" in it:
                    pv = it["pixel_values"]
                    pv = np.asarray(pv.cpu().numpy() if hasattr(pv, "cpu") else pv)
                    if pv.dtype != np.uint8 or pv.ndim != 5 or pv.shape[-1] != 3:
                        raise ValueError(f"pixel_values must be uint8 [n, T, H, W, 3], got {pv.dtype} {pv.shape}")
                    videos.extend(pv)
                elif isinstance(it, str) and "http" in it:
                    raise ValueError(f"Unsupported video content: {it} (downloading is Marqo's host code)")
                elif isinstance(it, str) or hasattr(it, "__fspath__"):
                    videos.append(_read_video_frames(it, self.arch["video_frames"]))
                else:
                    raise ValueError(f"Unsupported {modality.value} content type: {type(it)}, content: {it}")
            return self._encode_videos(videos, normalize)
        if modality == Modality.IMAGE and isinstance(content, (str, list)):
            first = content[0] if isinstance(content, list) else content
            if isinstance(first, str) and "http" not in first:   # the reference encodes such content as text
                return self.encode([first], modality=Modality.TEXT, normalize=normalize)
        if modality in (Modality.IMAGE, Modality.AUDIO):
            # the reference calls preprocessor(modality), which is None for a model without that tower
            raise TypeError(f"'NoneType' object is not callable: {self.model_properties.get('name')} has no "
                            f"{modality.value} tower")
        raise ValueError(f"Unsupported modality {modality}")


LOADERS = {
    model_registry.TYPE_OPEN_CLIP: B200OpenCLIP,
    model_registry.TYPE_HF: B200HuggingFace,
    model_registry.TYPE_HF_STELLA: B200HuggingFaceStella,
    model_registry.TYPE_CLIP: B200Clip,
    model_registry.TYPE_FP16_CLIP: B200Fp16Clip,
    model_registry.TYPE_MULTILINGUAL_CLIP: B200MultilingualClip,
    model_registry.TYPE_LANGUAGEBIND: B200LanguageBind,
}


def get_model_loader(model_name: Optional[str], model_properties: dict):
    """s2_inference.py:752-771"""
    model_type = model_properties['type']
    if model_type not in LOADERS:
        raise KeyError(f"model_name={model_name} for model_type={model_type} not in allowed model types")
    return LOADERS[model_type]


def register_with_marqo() -> None:
    """Install the engine's loader types into a live Marqo process (see INTEGRATION.md)."""
    from marqo.s2_inference import s2_inference as marqo_s2  # type: ignore
    marqo_s2.MODEL_PROPERTIES['loaders'].update(LOADERS)
    marqo_s2.MODEL_PROPERTIES['models'].update(model_registry.served_models())
