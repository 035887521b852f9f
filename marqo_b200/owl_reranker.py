"""The image reranker's model on the GPU: OWL-ViT detectors behind the `ReRankerOwl` name Marqo's reranker builds.

A search with `reRanker` set to an "owl/..." name reranks its image hits with `ReRankerOwl`
(reranking/rerank.py:32-45): each hit's image is loaded and resized by Pillow to 240 x 240 (`_load_image`), then
transformers' fp32 `OwlViTForObjectDetection` scores it against the query one image at a time
(reranking/cross_encoders.py:396-461), and `processor.post_process` turns every patch's logit and box into a score and a
corner box in 240-pixel coordinates.  `B200OwlDetector.detect` is that model and post-processing for all the hits in
one engine call (`Encoder.detect_images_u8`): the squash to the model's image size, the CLIP ViT trunk, the detection
heads and the 16-token CLIP text tower run on the GPU.

`register_with_marqo()` replaces the `ReRankerOwl` name rerank.py looks up with a factory: the names of
`model_registry.OWL_VIT_MODELS` on a CUDA device get a subclass of Marqo's own `ReRankerOwl` whose `load_model` caches a
`B200OwlDetector` in Marqo's model cache and whose `rerank` makes one `detect` call where the reference loops over the
hits; every other call gets the original class.  Everything else (the image loading and its cache, the sort, the
top-k, the box rescale, the DataFrame merge and the reranked results) is the reference's own code."""
from __future__ import annotations

import datetime
import os
from collections import defaultdict
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import model_registry, weights as weights_mod
from .cross_encoder import _cuda_index, _snapshot_dir
from .tokenizers import ClipBpeTokenizer

OWL_CONTEXT = 16   # OwlViTTextConfig.max_position_embeddings: the processor pads every query to 16 ids with "!" (0)


def query_ids(tokenizer: ClipBpeTokenizer, query: str) -> np.ndarray:
    """The query as OwlViTProcessor tokenises it: <start> BPE <end>, padded with 0 to 16 ids.  A query of more than 16
    ids is refused (ValueError), as the reference's 16-row position table refuses it."""
    ids = tokenizer([query], context_length=OWL_CONTEXT + 1)[0]
    if ids[OWL_CONTEXT] != 0:
        raise ValueError(f"query {query!r} is longer than OWL-ViT's {OWL_CONTEXT} tokens")
    return ids[:OWL_CONTEXT].astype(np.int32)


class B200OwlDetector:
    """OwlViTForObjectDetection (verify) with one text query per call, on one GPU.

    Weights and merges come from `weights` (a state dict under OwlViTForObjectDetection's names, or a path to one) or
    `random_init` (a seed, with the registry's shapes) together with `merges_file`; otherwise from the checkpoint's
    local snapshot directory (merges.txt, model.safetensors or pytorch_model.bin).  Nothing is downloaded."""

    def __init__(self, model_name: str, device=None, weights=None, random_init: Optional[int] = None,
                 merges_file=None, max_batch: int = 32):
        index = _cuda_index(device)
        if index is None:
            raise ValueError(f"B200OwlDetector runs on a CUDA device, not {device!r} (there is no CPU fallback)")
        entry = model_registry.OWL_VIT_MODELS.get(model_name)
        if entry is None:
            raise ValueError(f"{model_name} is not a served OWL-ViT model: {sorted(model_registry.OWL_VIT_MODELS)}")
        arch = entry["arch"]
        if weights is None and random_init is None:
            root = _snapshot_dir(entry["checkpoint"])
            merges_file = merges_file or os.path.join(root, "merges.txt")
            for fn in ("model.safetensors", "pytorch_model.bin"):
                if os.path.exists(os.path.join(root, fn)):
                    weights = os.path.join(root, fn)
                    break
            else:
                raise OSError(f"{root}: no model.safetensors or pytorch_model.bin")
        if weights is None:
            weights = weights_mod.random_owlvit_weights(arch, int(random_init))
        elif isinstance(weights, (str, os.PathLike)):
            weights = weights_mod.load_state_dict(str(weights))
        if merges_file is None:
            raise ValueError(f"{model_name}: `merges_file` (merges.txt) is needed with `weights` / `random_init`")
        from .engine import Encoder
        self.model_name = model_name
        self.image_size = int(arch["vision"]["image_size"])
        self.tokenizer = ClipBpeTokenizer(merges_file, context_length=OWL_CONTEXT)
        self.encoder = Encoder("clip", arch, weights_mod.owlvit_state_dict_to_engine(weights), device=index,
                               max_batch=max_batch)

    def close(self) -> None:
        enc, self.encoder = getattr(self, "encoder", None), None
        if enc is not None:
            enc.close()

    def query_ids(self, query: str) -> np.ndarray:
        return query_ids(self.tokenizer, query)

    def detect_raw(self, query: str, images) -> Tuple[np.ndarray, np.ndarray]:
        """logits fp32 [n, G^2] and pred_boxes fp32 [n, G^2, 4] (cx, cy, w, h) of n same-size images (PIL images or
        uint8 HWC arrays) against `query`."""
        if self.encoder is None:
            raise RuntimeError("B200OwlDetector is closed")
        hwc = np.stack([np.asarray(im.convert("RGB") if hasattr(im, "convert") else im, dtype=np.uint8)
                        for im in images])
        return self.encoder.detect_images_u8(hwc, self.query_ids(query))

    def detect(self, query: str, images) -> List[Tuple["object", "object"]]:
        """Per image (scores [G^2], corner boxes [G^2, 4]) as torch tensors: what the reference's
        `processor.post_process(outputs, target_sizes=[(h, w)])` gives, unthresholded, for images of h x w pixels
        (Marqo's 240 x 240): scores = sigmoid(logit), boxes = (cx - w/2, cy - h/2, cx + w/2, cy + h/2) scaled by the
        image's width and height."""
        import torch
        logits, boxes = self.detect_raw(query, images)
        out = []
        for i, im in enumerate(images):
            w, h = im.size if hasattr(im, "size") and not isinstance(im, np.ndarray) else (im.shape[1], im.shape[0])
            lg, bx = torch.from_numpy(logits[i]), torch.from_numpy(boxes[i])
            scores = torch.sigmoid(lg)
            cx, cy, bw, bh = bx.unbind(-1)
            corners = torch.stack([cx - 0.5 * bw, cy - 0.5 * bh, cx + 0.5 * bw, cy + 0.5 * bh], dim=-1)
            scale = torch.tensor([w, h, w, h], dtype=torch.float32)
            out.append((scores, corners * scale[None, :]))
        return out


def make_owl_reranker_class(original, cross_encoders, model_utils, detector=B200OwlDetector):
    """A subclass of Marqo's `ReRankerOwl` (`original`) that runs its model in the engine.  cross_encoders and
    model_utils are the modules the reference's rerank loop and model cache live in (Marqo's
    reranking.cross_encoders and reranking.model_utils, or stand-ins)."""
    cx, mu = cross_encoders, model_utils

    class B200ReRankerOwl(original):
        def load_model(self):
            """The detector of the remapped name, from Marqo's model cache under load_owl_vit's key, or built and
            cached there."""
            self._remapped_name = self._model_map[self.model_name]
            key = mu._create_model_cache_key(self._remapped_name, self.device)
            cache = mu.get_available_models()
            hit = cache.get(key)
            if hit is not None and isinstance(hit[mu.AvailableModelsKey.model], detector):
                self.model = hit[mu.AvailableModelsKey.model]
            else:
                self.model = detector(self._remapped_name, device=self.device)
                cache[key] = {mu.AvailableModelsKey.model: self.model,
                              mu.AvailableModelsKey.most_recently_used_time: datetime.datetime.now()}
            self.processor = None

        def rerank(self, query: str, results, image_attributes: List, num_highlights: int = 1):
            """ReRankerOwl.rerank with its per-image model loop replaced by one detect call per distinct query (one,
            in a search); the per-image sort, top-k, rescale and the merge are the reference's."""
            self.results = results
            self.image_attributes = image_attributes
            self.num_highlights = num_highlights
            if not isinstance(results, (dict, defaultdict)):
                raise TypeError(f"expected a dict or defaultdict, received {type(results)}")
            if len(results[cx.ResultsFields.hits]) == 0:
                cx.logger.warning("empty results for re-ranking. returning doing nothing...")
                return
            if self.model is None:
                self.load_model()
            self.format_results(results, searchable_fields=image_attributes)
            self.inputs_df = self.formatted_results.format_for_model(self.formatted_results.results_df,
                                                                     self.image_attributes, query=query)
            self.model_inputs = self._prepare_inputs(self.inputs_df)
            queries, image_names = zip(*self.model_inputs)
            self.images, self.original_sizes = self.load_images(image_names, self.image_size)
            detections: list = [None] * len(self.images)
            for q in dict.fromkeys(queries):
                idx = [i for i, qi in enumerate(queries) if qi == q]
                for i, det in zip(idx, self.model.detect(q, [self.images[i] for i in idx])):
                    detections[i] = det
            import torch
            _b, _s, _i, _bo = [], [], [], []
            for (scores, boxes), content, orig_size in zip(detections, image_names, self.original_sizes):
                labels = torch.zeros(scores.shape, dtype=torch.int64)
                boxes, scores, identifier = cx._process_owl_result([{"scores": scores, "labels": labels,
                                                                     "boxes": boxes}], content)
                boxes, scores, identifier = cx.sort_owl_boxes_scores(boxes, scores, identifier)
                boxes, scores, identifier = (cx._keep_top_k(boxes, k=num_highlights),
                                             cx._keep_top_k(scores, k=num_highlights),
                                             cx._keep_top_k(identifier, k=num_highlights))
                _bo += [list(cx.image_processor.rescale_box(b.detach().cpu().tolist(), self.image_size, orig_size))
                        for b in boxes]
                _b.append(boxes)
                _s.append(scores)
                _i += identifier
            self.boxes_original = _bo
            self.boxes = torch.cat(_b)
            self.scores = torch.cat(_s)
            self.identifier = _i
            Columns, ResultsFields = cx.Columns, cx.ResultsFields
            self.boxes_scores_df = cx.pd.DataFrame(
                zip(self.boxes.detach().cpu().tolist(), self.scores.detach().cpu().tolist(), self.identifier,
                    self.boxes_original),
                columns=[Columns.bbox, ResultsFields.reranker_score, Columns.field_content, Columns.bbox_original])
            self.inputs_df = self.boxes_scores_df.merge(self.inputs_df, left_on=Columns.field_content,
                                                        right_on=Columns.field_content)
            self.get_reranked_results(highlight_content_column=Columns.bbox_original)

    B200ReRankerOwl.__name__ = B200ReRankerOwl.__qualname__ = "B200ReRankerOwl"
    return B200ReRankerOwl


def make_owl_factory(original, served):
    """A stand-in for the `ReRankerOwl` class: `served` for the names of OWL_VIT_MODELS on a CUDA device, `original`
    for every other name or device, with the caller's arguments."""
    def factory(*args, **kwargs):
        kw = dict(zip(("model_name", "device", "image_size"), args))   # ReRankerOwl's positional order
        kw.update(kwargs)
        if kw.get("model_name") in model_registry.OWL_VIT_MODELS and _cuda_index(kw.get("device")) is not None:
            return served(*args, **kwargs)
        return original(*args, **kwargs)

    factory.original = original
    factory.served = served
    return factory


def register_with_marqo() -> None:
    """Serve Marqo's image reranker on the GPU: replace the ReRankerOwl that reranking/rerank.py calls with the factory
    above (see INTEGRATION.md).  Calling it again keeps the first original."""
    from marqo.s2_inference.reranking import cross_encoders, model_utils, rerank  # type: ignore
    original = getattr(rerank.ReRankerOwl, "original", rerank.ReRankerOwl)
    rerank.ReRankerOwl = make_owl_factory(original, make_owl_reranker_class(original, cross_encoders, model_utils))
