"""add_documents fast path (SURVEY §8 cfg3 / VERDICT r01 "missing #2"): embeddings go from the encoder's projection +
L2 epilogue straight into the GPU row store — `List[List[float]]` is never built, no per-document device call.

Shape of the reference flow this sits in (one request = one batch of documents):
  AddDocumentsHandler.add_documents (src/marqo/core/vespa_index/add_documents_handler.py:123-177)
    -> tensor_fields_container collects (key, content) chunks per field type
    -> BatchCachingVectoriser vectorises ALL chunks of a modality in one call and serves them back by key
       (src/marqo/core/inference/tensor_fields_container.py:196-223)
    -> SemiStructuredVespaDocument puts {str(i): embeddings[i]} under `marqo__embeddings_<field>`
       (src/marqo/core/semi_structured_vespa_index/semi_structured_document.py:139-141)
    -> vespa_client.feed_batch(vespa_docs, schema)                                   (add_documents_handler.py:177)
Here `DeviceBatchVectoriser` is the BatchCachingVectoriser whose cache is one CUDA tensor, and a document's
`marqo__embeddings_<field>` is a `DeviceChunks` view of it; GpuTensorIndex.feed_batch appends a whole batch's rows per
tensor field with ONE b200_index_add_device_docs call.
"""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Sequence, Tuple

from .gpu_tensor_index import CHUNKS_PREFIX, EMBEDDINGS_PREFIX, DeviceChunks, GpuTensorIndex


class DeviceBatchVectoriser:
    """BatchCachingVectoriser (tensor_fields_container.py:196-223) with the embedding cache resident on the GPU.
    `chunks_to_vectorise`: [(key, content)] with keys '<prefix>_<i>' — the reference's key scheme; content is whatever
    the model's encode_to_device accepts for that modality."""

    def __init__(self, model, chunks_to_vectorise: Sequence[Tuple[str, Any]], normalize_embeddings: bool = True,
                 default: str = "text", contents_array=None, **encode_kwargs):
        self.index: Dict[str, int] = {key: i for i, (key, _) in enumerate(chunks_to_vectorise)}
        if not chunks_to_vectorise:
            self.embeddings = None
            return
        contents = contents_array if contents_array is not None else [c for _, c in chunks_to_vectorise]
        kw = dict(encode_kwargs)
        if hasattr(model, "encode_image"):      # CLIP-type loader: routing argument of abstract_clip_model.py:56-75
            kw["default"] = default
        self.embeddings = model.encode_to_device(contents, normalize=normalize_embeddings, **kw)   # CUDA fp32 [n, dim]

    def vectorise(self, content_chunks: Sequence[Any], key_prefix: str) -> DeviceChunks:
        """The chunks '<key_prefix>_0' .. '<key_prefix>_<n-1>' as one DeviceChunks (they are consecutive rows)."""
        n = len(content_chunks)
        first = self.index[f"{key_prefix}_0"]
        for i in range(1, n):
            if self.index[f"{key_prefix}_{i}"] != first + i:
                raise ValueError(f"chunks of {key_prefix} are not consecutive in the vectorised batch")
        e = self.embeddings
        return DeviceChunks([str(i) for i in range(n)], e[first:first + n].data_ptr(), int(e.shape[1]), owner=e)


def add_documents_device(index: GpuTensorIndex, schema: str, docs: Sequence[Dict[str, Any]],
                         tensor_fields: Dict[str, Tuple[Any, str]], normalize_embeddings: bool = True,
                         id_field: str = "_id", device_contents: Optional[Dict[str, Any]] = None):
    """One add_documents batch on the fast path.

    docs: Marqo documents ({'_id': ..., field: content, ...}); `tensor_fields` maps a tensor field name to
    (model loader object, 'image' | 'text').  Every tensor field is vectorised in ONE encode_to_device call over the
    batch (one chunk per document and field: images are not patch-chunked, captions are single chunks — the cfg3
    shape), the embeddings stay in HBM, and the batch is fed with one feed_batch.
    `device_contents[field]`: optional pre-assembled batch content for the field (a uint8 [n, H, W, 3] CUDA tensor, a
    list of n uint8 [H_i, W_i, 3] CUDA tensors of any sizes such as decode_images_to_device returns, or an int32
    [n, seq] token-id array) replacing the per-document contents — what a loader that decodes / tokenises in bulk
    hands over.  Returns feed_batch's FeedBatchResponse."""
    vectorisers: Dict[str, DeviceBatchVectoriser] = {}
    for field, (model, modality) in tensor_fields.items():
        chunks = [(f"{doc.get(id_field, i)}_{field}_0", doc.get(field)) for i, doc in enumerate(docs)]
        contents = None if device_contents is None else device_contents.get(field)
        if contents is not None and not isinstance(contents, list) and hasattr(contents, "shape") and \
                getattr(contents, "ndim", 0) == 4:
            contents = list(contents)       # a stacked image batch: the loader re-stacks device tensors without copies
        vectorisers[field] = DeviceBatchVectoriser(model, chunks, normalize_embeddings, default=modality,
                                                   contents_array=contents)
    batch = []
    for i, doc in enumerate(docs):
        doc_id = str(doc.get(id_field, i))
        fields: Dict[str, Any] = {"marqo__id": doc_id}
        for k, v in doc.items():
            if k == id_field or k in tensor_fields:
                continue
            fields[k] = v
        for field in tensor_fields:
            content = doc.get(field)
            fields[f"{CHUNKS_PREFIX}_{field}"] = [content if isinstance(content, str) else f"{field}::{doc_id}"]
            fields[f"{EMBEDDINGS_PREFIX}_{field}"] = vectorisers[field].vectorise([content], f"{doc.get(id_field, i)}_{field}")
        batch.append({"id": doc_id, "fields": fields})
    return index.feed_batch(batch, schema)
