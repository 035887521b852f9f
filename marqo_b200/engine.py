"""Thin Python objects over the C ABI handles (include/marqo_b200.h).  No arithmetic happens here."""
from __future__ import annotations

import ctypes as C
import threading
from typing import Optional, Sequence, Tuple

import numpy as np

from . import _native as N

_METRICS = {
    # names: src/marqo/core/models/marqo_index.py:63-69 (DistanceMetric)
    "prenormalized-angular": N.METRIC_PRENORMALIZED_ANGULAR,
    "angular": N.METRIC_ANGULAR,
    "dotproduct": N.METRIC_DOTPRODUCT,
    "euclidean": N.METRIC_EUCLIDEAN,
}


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _as(a, dtype) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=dtype)


class RowStore:
    """GPU-resident fp16 embedding matrix with exact top-k search (b200_index_*)."""

    def __init__(self, dim: int, metric: str = "prenormalized-angular", device: int = 0, capacity: int = 0,
                 _handle=None):
        self._lib = N.load()
        self.dim = int(dim)
        self.metric = metric
        self.device = int(device)
        if _handle is not None:
            self._h = _handle
            return
        if metric not in _METRICS:
            raise ValueError(f"unknown distance metric {metric!r}; expected one of {sorted(_METRICS)}")
        h = C.c_void_p()
        N.check(self._lib.b200_index_create(self.device, self.dim, _METRICS[metric], int(capacity), C.byref(h)))
        self._h = h

    # -- lifetime -------------------------------------------------------------------------------
    def close(self) -> None:
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._lib.b200_index_destroy(h)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _handle(self):
        if not self._h:
            raise RuntimeError("RowStore is closed")
        return self._h

    # -- mutation -------------------------------------------------------------------------------
    def add(self, vecs, doc_ids: Optional[Sequence[int]] = None) -> None:
        v = _as(vecs, np.float32)
        if v.ndim != 2 or v.shape[1] != self.dim:
            raise ValueError(f"expected [m, {self.dim}] embeddings, got {v.shape}")
        d = None
        if doc_ids is not None:
            d = _as(doc_ids, np.int32)
            if d.shape != (v.shape[0],):
                raise ValueError("doc_ids must have one entry per row")
        N.check(self._lib.b200_index_add(self._handle(), _ptr(v), _ptr(d), v.shape[0]))

    def add_device(self, d_vecs_ptr: int, m: int, d_doc_ids_ptr: Optional[int] = None) -> None:
        N.check(self._lib.b200_index_add_device(self._handle(), C.c_void_p(d_vecs_ptr),
                                                C.c_void_p(d_doc_ids_ptr) if d_doc_ids_ptr else None, int(m)))

    def add_device_docs(self, d_vecs_ptr: int, doc_ids: Sequence[int]) -> None:
        """Embeddings already on the device (fp32 [m, dim]), document numbers on the host: the add_documents fast path."""
        d = _as(doc_ids, np.int32)
        N.check(self._lib.b200_index_add_device_docs(self._handle(), C.c_void_p(d_vecs_ptr), _ptr(d), d.shape[0]))

    def delete_doc(self, doc_id: int) -> None:
        N.check(self._lib.b200_index_delete_doc(self._handle(), int(doc_id)))

    def delete_rows(self, rows: Sequence[int]) -> None:
        r = _as(rows, np.int32)
        N.check(self._lib.b200_index_delete_rows(self._handle(), _ptr(r), r.shape[0]))

    def compact(self) -> np.ndarray:
        """Squeeze tombstoned rows out; -> new_of_old int32 [old rows] (-1 = removed)."""
        n = len(self)
        m = np.empty(n, np.int32)
        left = C.c_int64(0)
        N.check(self._lib.b200_index_compact(self._handle(), _ptr(m), C.byref(left)))
        return m

    # -- queries --------------------------------------------------------------------------------
    def __len__(self) -> int:
        n = C.c_int64(0)
        N.check(self._lib.b200_index_num_rows(self._handle(), C.byref(n)))
        return n.value

    def get_row(self, row: int) -> np.ndarray:
        out = np.empty(self.dim, dtype=np.float32)
        N.check(self._lib.b200_index_get_row(self._handle(), int(row), _ptr(out)))
        return out

    def get_rows(self, rows: Sequence[int]) -> np.ndarray:
        r = _as(rows, np.int64)
        out = np.empty((r.shape[0], self.dim), dtype=np.float32)
        N.check(self._lib.b200_index_get_rows(self._handle(), _ptr(r), r.shape[0], _ptr(out)))
        return out

    def search(self, queries, k: int, mult: Sequence[Tuple[int, float]] = (), add: Sequence[Tuple[int, float]] = (),
               filter_bits: Optional[np.ndarray] = None, filter_docs: int = 0,
               filter_tag: int = 0) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """-> (doc [nq,k] int32, row [nq,k] int32, score [nq,k] float64); unused slots are -1/-1/-inf.
        mult / add: score modifiers [(attribute column, weight), ...] (score = modified score then);
        filter_bits: uint32 bitset over document numbers (bit set = may match), covering filter_docs documents;
        filter_tag != 0 lets the device keep the bitset between calls."""
        q = _as(queries, np.float32)
        if q.ndim == 1:
            q = q[None, :]
        if q.ndim != 2 or q.shape[1] != self.dim:
            raise ValueError(f"expected [nq, {self.dim}] queries, got {q.shape}")
        nq = q.shape[0]
        doc = np.empty((nq, k), dtype=np.int32)
        row = np.empty((nq, k), dtype=np.int32)
        score = np.empty((nq, k), dtype=np.float64)
        opts = None
        keep = []
        if mult or add or filter_bits is not None:
            o = N.SearchOpts()
            mc = _as([c for c, _ in mult], np.int32)
            mw = _as([w for _, w in mult], np.float64)
            ac = _as([c for c, _ in add], np.int32)
            aw = _as([w for _, w in add], np.float64)
            keep = [mc, mw, ac, aw]
            o.mult_cols, o.mult_w, o.n_mult = mc.ctypes.data, mw.ctypes.data, len(mc)
            o.add_cols, o.add_w, o.n_add = ac.ctypes.data, aw.ctypes.data, len(ac)
            if filter_bits is not None:
                fb = _as(filter_bits, np.uint32)
                if fb.shape[0] * 32 < filter_docs:
                    raise ValueError("filter_bits does not cover filter_docs documents")
                keep.append(fb)
                o.filter_bits, o.filter_docs, o.filter_tag = fb.ctypes.data, int(filter_docs), int(filter_tag)
            opts = C.byref(o)
        N.check(self._lib.b200_index_search_ex(self._handle(), _ptr(q), nq, int(k), opts, _ptr(doc), _ptr(row),
                                               _ptr(score)))
        del keep
        return doc, row, score

    def search_stats(self) -> dict:
        a, b, c, d = C.c_int64(0), C.c_int64(0), C.c_int64(0), C.c_int64(0)
        N.check(self._lib.b200_index_search_stats(self._handle(), C.byref(a), C.byref(b), C.byref(c), C.byref(d)))
        return {"groups": a.value, "flagged": b.value, "collect_passes": c.value, "unresolved_async": d.value}

    # -- score modifiers -----------------------------------------------------------------------
    def set_attributes(self, column: int, doc_ids: Sequence[int], values: Optional[Sequence[float]]) -> None:
        """Set (values given) or remove (values None) the numeric attribute `column` of the listed documents;
        column == -1 with values None removes every attribute of those documents."""
        d = _as(doc_ids, np.int32)
        v = None
        if values is not None:
            v = _as(values, np.float64)
            if v.shape != d.shape:
                raise ValueError("values must have one entry per document")
        N.check(self._lib.b200_index_set_attributes(self._handle(), int(column), _ptr(d), _ptr(v), d.shape[0]))

    def set_attributes_multi(self, columns: Sequence[int], doc_ids: Sequence[int], values: Sequence[float]) -> None:
        """Many (column, document, value) cells in one call."""
        c, d, v = _as(columns, np.int32), _as(doc_ids, np.int32), _as(values, np.float64)
        if not (c.shape == d.shape == v.shape):
            raise ValueError("columns, doc_ids and values must have the same length")
        N.check(self._lib.b200_index_set_attributes_multi(self._handle(), _ptr(c), _ptr(d), _ptr(v), c.shape[0]))

    def search_modified(self, queries, k: int, mult: Sequence[Tuple[int, float]] = (),
                        add: Sequence[Tuple[int, float]] = ()) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """search() ranked by modify(closeness) = prod(w * attr) * closeness + sum(w * attr)
        (unstructured_vespa_schema.py:266-271).  mult / add: [(attribute column, weight), ...].
        -> (doc, row, modified score)."""
        return self.search(queries, k, mult=mult, add=add)

    def search_device(self, d_q_ptr: int, nq: int, k: int, d_doc_ptr: int, d_row_ptr: int, d_score_ptr: int,
                      sync: bool = True) -> None:
        N.check(self._lib.b200_index_search_device(self._handle(), C.c_void_p(d_q_ptr), int(nq), int(k),
                                                   C.c_void_p(d_doc_ptr), C.c_void_p(d_row_ptr),
                                                   C.c_void_p(d_score_ptr), 1 if sync else 0))

    def set_stream(self, cuda_stream: Optional[int]) -> None:
        """cuda_stream: a cudaStream_t handle (0 = legacy default stream); None restores the private stream."""
        N.check(self._lib.b200_index_set_stream(self._handle(), C.c_void_p(cuda_stream or 0),
                                                0 if cuda_stream is None else 1))

    def set_doc_offset(self, offset: int) -> None:
        N.check(self._lib.b200_index_set_doc_offset(self._handle(), int(offset)))

    def merge_shards_device(self, d_gathered_ptr: int, nshards: int, nq: int, k: int, d_doc_ptr: int, d_row_ptr: int,
                            d_score_ptr: int, sync: bool = True) -> None:
        N.check(self._lib.b200_topk_merge_device(self._handle(), C.c_void_p(d_gathered_ptr), nshards, nq, k,
                                                 C.c_void_p(d_doc_ptr), C.c_void_p(d_row_ptr), C.c_void_p(d_score_ptr),
                                                 1 if sync else 0))

    def search_exchange(self, exchange: "Exchange", d_q_ptr: int, nq: int, k: int, d_block_ptr: int, d_doc_ptr: int,
                        d_row_ptr: int, d_score_ptr: int, sync: bool = True) -> None:
        """Local search + fused peer-store exchange + merge (b200_index_search_exchange)."""
        N.check(self._lib.b200_index_search_exchange(self._handle(), exchange._handle(), C.c_void_p(d_q_ptr), int(nq),
                                                     int(k), C.c_void_p(d_block_ptr), C.c_void_p(d_doc_ptr),
                                                     C.c_void_p(d_row_ptr), C.c_void_p(d_score_ptr), 1 if sync else 0))

    def last_timing(self) -> Tuple[float, float]:
        a, b = C.c_float(0), C.c_float(0)
        N.check(self._lib.b200_index_last_timing(self._handle(), C.byref(a), C.byref(b)))
        return a.value, b.value

    # -- persistence ----------------------------------------------------------------------------
    def save(self, path: str) -> None:
        N.check(self._lib.b200_index_save(self._handle(), str(path).encode()))

    @classmethod
    def load(cls, path: str, device: int = 0) -> "RowStore":
        lib = N.load()
        h = C.c_void_p()
        N.check(lib.b200_index_load(int(device), str(path).encode(), C.byref(h)))
        d, m, dev = C.c_int(0), C.c_int(0), C.c_int(0)
        N.check(lib.b200_index_info(h, C.byref(d), C.byref(m), C.byref(dev)))
        names = {v: k for k, v in _METRICS.items()}
        return cls(dim=d.value, metric=names[m.value], device=dev.value, _handle=h)


class Exchange:
    """Symmetric NVLink exchange buffer of one rank (b200_exchange_*).  `handle` (64 bytes) is what the ranks swap;
    `open(all_handles)` maps the peers' buffers."""

    def __init__(self, device: int, rank: int, world: int, max_nq: int = 64, max_k: int = 16):
        self._lib = N.load()
        h = C.c_void_p()
        buf = (C.c_uint8 * N.EXCHANGE_HANDLE_BYTES)()
        N.check(self._lib.b200_exchange_create(int(device), int(rank), int(world), int(max_nq), int(max_k), C.byref(h),
                                               C.cast(buf, C.c_void_p)))
        self._h = h
        self.rank, self.world = int(rank), int(world)
        self.handle = bytes(buf)

    def open(self, handles: Sequence[bytes]) -> None:
        if len(handles) != self.world or any(len(h) != N.EXCHANGE_HANDLE_BYTES for h in handles):
            raise ValueError("expected one 64-byte handle per rank")
        blob = b"".join(handles)
        N.check(self._lib.b200_exchange_open(self._handle(), C.c_char_p(blob)))

    def _handle(self):
        if not self._h:
            raise RuntimeError("Exchange is closed")
        return self._h

    def close(self) -> None:
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._lib.b200_exchange_destroy(h)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def topk_merge(doc: np.ndarray, row: np.ndarray, score: np.ndarray) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Merge per-shard lists [nshards, nq, k] into [nq, k] under (score desc, doc asc)."""
    doc, row, score = _as(doc, np.int32), _as(row, np.int32), _as(score, np.float64)
    ns, nq, k = doc.shape
    od = np.empty((nq, k), np.int32)
    orow = np.empty((nq, k), np.int32)
    osc = np.empty((nq, k), np.float64)
    N.check(N.load().b200_topk_merge(ns, nq, k, _ptr(doc), _ptr(row), _ptr(score), _ptr(od), _ptr(orow), _ptr(osc)))
    return od, orow, osc


# ---------------------------------------------------------------------------------------------------------
# Encoders (b200_model_*)
# ---------------------------------------------------------------------------------------------------------
def _to_numpy_f32(t) -> np.ndarray:
    if hasattr(t, "detach"):
        t = t.detach().to("cpu").float().numpy()
    return np.ascontiguousarray(t, dtype=np.float32)


class Encoder:
    """A CLIP, ResNet CLIP, ConvNeXt CLIP, EVA02 CLIP or SigLIP (vision + text towers), BERT, MPNet, XLM-R or GTE
    encoder resident on one GPU.

    `config` keys — CLIP: embed_dim, act ("gelu"|"quickgelu"), mean, std, resize_mode (optional: "squash" resizes
    images of another size without a crop), vision{width,layers,heads,mlp,patch,image_size},
    text{width,layers,heads,mlp,ctx,vocab}; CoCa is CLIP with vision.attn_pool_heads (its attentional pooler) and
    text.embed_cls (its appended CLS row; ctx counts it, so the ids are ctx - 1 wide); OWL-ViT is CLIP with
    owl_detect (the detection head in place of visual.proj, run by detect_images_u8); LanguageBind's video model is CLIP
    with video_frames (the vision tower a video tower, run by encode_videos_u8);  SigLIP: the CLIP keys plus ln_eps (embed_dim == vision
    width);  ResNet CLIP ("clip_resnet"): embed_dim, act, mean, std, the text tower's width, layers, heads, mlp, ctx,
    vocab at the top level (layers 0: no text tower), resnet{layers [4], width, heads, image_size} (None: no image
    tower);  ConvNeXt CLIP ("clip_convnext"): the ResNet CLIP keys with convnext{dims [4], depths [4], image_size,
    ln_eps, head ("linear"|"mlp")} (None: no image tower) in place of resnet;  EVA02 CLIP ("clip_eva"): the ResNet
    CLIP keys with eva{width, layers, heads, mlp (the SwiGLU hidden size), patch, image_size, ln_eps, rope_ref_grid}
    (None: no image tower) in place of resnet;  BERT: width, layers, heads, mlp, vocab,
    max_pos, type_vocab,
    pool ("mean"|"cls"), proj_dim (optional: M-CLIP's projected text head of that many outputs, whose weights are
    LinearTransformation.weight [proj_dim, width] and .bias), num_labels (optional: a BertForSequenceClassification
    cross-encoder of that many labels, run by classify_tokens, whose weights add pooler.dense.* and classifier.*);  MPNet: width, layers, heads, mlp, vocab, max_pos (max_position_embeddings: sequences of up to
    max_pos - pad_id - 1 tokens), pad_id, ln_eps, rel_buckets, rel_max_distance, pool;  XLM-R: width, layers, heads,
    mlp, vocab, max_pos (as MPNet), pad_id, ln_eps, pool, proj_dim (as BERT);  GTE (NewModel: the Stella embedders): width, layers, heads,
    mlp (the GeGLU hidden size), vocab, type_vocab, ctx, ln_eps, rope_theta, rope_ntk_factor, pool.  `weights` maps
    checkpoint parameter names (open_clip state_dict names / HF BertModel / MPNetModel / XLMRobertaModel / NewModel
    names) to fp32 arrays or torch tensors.
    """

    def __init__(self, arch: str, config: dict, weights: dict, device: int = 0, max_batch: int = 256):
        self._lib = N.load()
        self.arch = arch
        self.device = int(device)
        d = N.ModelDesc()
        d.max_batch = int(max_batch)
        if arch in ("clip", "siglip"):
            d.arch = N.ARCH_CLIP if arch == "clip" else N.ARCH_SIGLIP
            if arch == "siglip":
                d.layer_norm_eps = float(config["ln_eps"])
            d.embed_dim = int(config["embed_dim"])
            d.act = N.ACT_QUICKGELU if config.get("act", "gelu") == "quickgelu" else N.ACT_GELU
            mean = config.get("mean", (0.48145466, 0.4578275, 0.40821073))
            std = config.get("std", (0.26862954, 0.26130258, 0.27577711))
            for i in range(3):
                d.image_mean[i] = float(np.float32(mean[i]))
                d.image_std[i] = float(np.float32(std[i]))
            v, t = config.get("vision"), config.get("text")
            if v:
                d.vision = N.TowerDesc(v["width"], v["layers"], v["heads"], v["mlp"], 0, 0, v.get("image_size", 224),
                                       v["patch"])
                d.attn_pool_heads = int(v.get("attn_pool_heads", 0))
            if t:
                d.text = N.TowerDesc(t["width"], t["layers"], t["heads"], t["mlp"], t["ctx"], t["vocab"], 0, 0)
                d.text_embed_cls = int(bool(t.get("embed_cls", False)))
            # open_clip's resize_mode "squash" (SigLIP, the DFN5B CLIP models): the GPU resize scales x and y to
            # image_size independently instead of cropping
            d.resize_squash = int(config.get("resize_mode") == "squash")
            d.owl_detect = int(bool(config.get("owl_detect", False)))
            # LanguageBind's video model: the vision tower runs over video_frames frames with its temporal layers
            d.video_frames = int(config.get("video_frames") or 0)
            self.video_frames = int(d.video_frames)
            self.image_size = v.get("image_size", 224) if v else 0
            self.grid = self.image_size // v["patch"] if v else 0
        elif arch == "clip_resnet":
            d.arch = N.ARCH_CLIP_RESNET
            d.embed_dim = int(config["embed_dim"])
            d.act = N.ACT_QUICKGELU if config.get("act", "gelu") == "quickgelu" else N.ACT_GELU
            for i in range(3):
                d.image_mean[i] = float(np.float32(config["mean"][i]))
                d.image_std[i] = float(np.float32(config["std"][i]))
            r = config.get("resnet")
            if r:
                for i in range(4):
                    d.resnet_layers[i] = int(r["layers"][i])
                d.resnet_width, d.resnet_heads = int(r["width"]), int(r["heads"])
                d.resnet_image_size = int(r.get("image_size", 224))
            if config.get("layers"):
                d.text = N.TowerDesc(config["width"], config["layers"], config["heads"], config["mlp"], config["ctx"],
                                     config["vocab"], 0, 0)
            self.image_size = int(r.get("image_size", 224)) if r else 0
        elif arch == "clip_convnext":
            d.arch = N.ARCH_CLIP_CONVNEXT
            d.embed_dim = int(config["embed_dim"])
            d.act = N.ACT_QUICKGELU if config.get("act", "gelu") == "quickgelu" else N.ACT_GELU
            for i in range(3):
                d.image_mean[i] = float(np.float32(config["mean"][i]))
                d.image_std[i] = float(np.float32(config["std"][i]))
            cx = config.get("convnext")
            if cx:
                for i in range(4):
                    d.convnext_dims[i], d.convnext_depths[i] = int(cx["dims"][i]), int(cx["depths"][i])
                d.convnext_image_size = int(cx["image_size"])
                d.layer_norm_eps = float(cx["ln_eps"])
                d.convnext_head = {"linear": 0, "mlp": 1}[cx["head"]]
            if config.get("layers"):
                d.text = N.TowerDesc(config["width"], config["layers"], config["heads"], config["mlp"], config["ctx"],
                                     config["vocab"], 0, 0)
            self.image_size = int(cx["image_size"]) if cx else 0
        elif arch == "clip_eva":
            d.arch = N.ARCH_CLIP_EVA
            d.embed_dim = int(config["embed_dim"])
            d.act = N.ACT_QUICKGELU if config.get("act", "gelu") == "quickgelu" else N.ACT_GELU
            for i in range(3):
                d.image_mean[i] = float(np.float32(config["mean"][i]))
                d.image_std[i] = float(np.float32(config["std"][i]))
            ev = config.get("eva")
            if ev:
                d.vision = N.TowerDesc(ev["width"], ev["layers"], ev["heads"], ev["mlp"], 0, 0, ev["image_size"],
                                       ev["patch"])
                d.layer_norm_eps = float(ev["ln_eps"])
                d.eva_rope_ref_grid = int(ev["rope_ref_grid"])
            if config.get("layers"):
                d.text = N.TowerDesc(config["width"], config["layers"], config["heads"], config["mlp"], config["ctx"],
                                     config["vocab"], 0, 0)
            self.image_size = int(ev["image_size"]) if ev else 0
        elif arch == "bert":
            d.arch = N.ARCH_BERT
            d.cls_labels = int(config.get("num_labels") or 0)
            d.embed_dim = int(d.cls_labels or config.get("proj_dim") or config["width"])
            d.text_proj_dim = int(config.get("proj_dim") or 0)
            d.pool = N.POOL_CLS if config.get("pool", "mean") == "cls" else N.POOL_MEAN
            d.type_vocab = int(config.get("type_vocab", 2))
            d.text = N.TowerDesc(config["width"], config["layers"], config["heads"], config["mlp"],
                                 config.get("max_pos", 512), config["vocab"], 0, 0)
            self.image_size = 0
        elif arch == "xlmr":
            d.arch = N.ARCH_XLMR
            d.embed_dim = int(config.get("proj_dim") or config["width"])
            d.text_proj_dim = int(config.get("proj_dim") or 0)
            d.pool = N.POOL_CLS if config.get("pool", "mean") == "cls" else N.POOL_MEAN
            d.pad_id = int(config.get("pad_id", 1))
            d.layer_norm_eps = float(config["ln_eps"])
            ctx = int(config.get("max_pos", 514)) - d.pad_id - 1   # RoBERTa positions start after the pad id
            d.text = N.TowerDesc(config["width"], config["layers"], config["heads"], config["mlp"], ctx, config["vocab"],
                                 0, 0)
            self.image_size = 0
        elif arch == "mpnet":
            d.arch = N.ARCH_MPNET
            d.embed_dim = int(config["width"])
            d.pool = N.POOL_CLS if config.get("pool", "mean") == "cls" else N.POOL_MEAN
            d.pad_id = int(config.get("pad_id", 1))
            d.layer_norm_eps = float(config["ln_eps"])      # MPNetConfig's default (1e-12) is not the checkpoints' value
            d.rel_buckets = int(config.get("rel_buckets", 32))
            d.rel_max_distance = int(config.get("rel_max_distance", 128))
            ctx = int(config.get("max_pos", 514)) - d.pad_id - 1
            d.text = N.TowerDesc(config["width"], config["layers"], config["heads"], config["mlp"], ctx, config["vocab"],
                                 0, 0)
            self.image_size = 0
        elif arch == "gte":
            d.arch = N.ARCH_GTE
            d.embed_dim = int(config["width"])
            d.pool = N.POOL_CLS if config.get("pool", "mean") == "cls" else N.POOL_MEAN
            d.type_vocab = int(config.get("type_vocab", 2))
            d.layer_norm_eps = float(config["ln_eps"])
            d.rope_theta = float(config["rope_theta"])
            d.rope_ntk_factor = float(config["rope_ntk_factor"])
            d.text = N.TowerDesc(config["width"], config["layers"], config["heads"], config["mlp"], config["ctx"],
                                 config["vocab"], 0, 0)
            self.image_size = 0
        else:
            raise ValueError(f"unknown arch {arch!r}")
        self.embed_dim = int(d.embed_dim)
        self._stage_ptr, self._stage_bytes = None, 0
        self._stage_lock = threading.Lock()
        self._pool = None
        h = C.c_void_p()
        N.check(self._lib.b200_model_create(self.device, C.byref(d), C.byref(h)))
        self._h = h
        try:
            for name, t in weights.items():
                a = _to_numpy_f32(t)
                N.check(self._lib.b200_model_load_tensor(h, name.encode(), _ptr(a), a.size))
            N.check(self._lib.b200_model_finalize(h))
        except Exception:
            self.close()
            raise

    def close(self) -> None:
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._lib.b200_model_destroy(h)
        pool, self._pool = getattr(self, "_pool", None), None
        if pool is not None:
            pool.shutdown(wait=False)
        st, self._stage_ptr = getattr(self, "_stage_ptr", None), None
        if st:
            self._lib.b200_host_free(st)
            self._stage_bytes = 0

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _handle(self):
        if not self._h:
            raise RuntimeError("Encoder is closed")
        return self._h

    def _staging(self, nbytes: int) -> np.ndarray:
        """A reusable page-locked uint8 buffer of at least nbytes (caller holds self._stage_lock)."""
        if getattr(self, "_stage_bytes", 0) < nbytes:
            if getattr(self, "_stage_ptr", None):
                self._lib.b200_host_free(self._stage_ptr)
                self._stage_ptr, self._stage_bytes = None, 0
            want = int(nbytes * 1.25) + 4096
            p = C.c_void_p()
            N.check(self._lib.b200_host_alloc(want, C.byref(p)))
            self._stage_ptr, self._stage_bytes = p, want
        return np.ctypeslib.as_array((C.c_uint8 * self._stage_bytes).from_address(self._stage_ptr.value))

    def encode_images_u8_list(self, images: Sequence[np.ndarray], normalize: bool = True) -> np.ndarray:
        """uint8 HWC images of ONE size, given one by one (what Marqo's download threads hand over): they are
        assembled in a reusable page-locked staging buffer — no fresh 38 MB allocation per batch, full-rate H2D."""
        n = len(images)
        if n == 0:
            raise ValueError("expected at least one image")
        h, w = images[0].shape[:2]
        out = np.empty((n, self.embed_dim), np.float32)
        with self._stage_lock:
            buf = self._staging(n * h * w * 3)[: n * h * w * 3].reshape(n, h, w, 3)
            for i, a in enumerate(images):
                if a.shape != (h, w, 3) or a.dtype != np.uint8:
                    raise ValueError(f"image {i}: expected uint8 [{h}, {w}, 3], got {a.dtype} {a.shape}")

            self._fill(n, n * h * w * 3, lambda i: np.copyto(buf[i], images[i]))
            N.check(self._lib.b200_model_encode_images_u8(self._handle(), C.c_void_p(self._stage_ptr.value), n, h, w,
                                                          1 if normalize else 0, _ptr(out)))
        return out

    def _fill(self, n: int, nbytes: int, copy) -> None:
        """copy(i) for i < n: the staging copies of n images of nbytes in all (np.copyto releases the GIL for the
        memcpy), on eight threads from 8 MB up."""
        def fill(lo: int, hi: int) -> None:
            for i in range(lo, hi):
                copy(i)

        if nbytes >= (8 << 20):   # a 38 MB batch: ~4 ms on one core, < 1 ms on eight
            if self._pool is None:
                from concurrent.futures import ThreadPoolExecutor
                self._pool = ThreadPoolExecutor(8, thread_name_prefix="b200-stage")
            step = (n + 7) // 8
            list(self._pool.map(lambda lo: fill(lo, min(n, lo + step)), range(0, n, step)))
        else:
            fill(0, n)

    def encode_images_u8_ragged(self, images: Sequence[np.ndarray], normalize: bool = True) -> np.ndarray:
        """uint8 HWC images of any sizes, [h_i, w_i, 3] each, in one call: they are packed back to back into the
        page-locked staging buffer (one H2D copy per sub-batch), resized together on the GPU and encoded in one tower
        pass per sub-batch.  Row i of the result is image i's embedding."""
        n = len(images)
        if n == 0:
            raise ValueError("expected at least one image")
        for i, a in enumerate(images):
            if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3:
                raise ValueError(f"image {i}: expected uint8 [H, W, 3], got {a.dtype} {a.shape}")
        sizes = [a.shape[0] * a.shape[1] * 3 for a in images]
        offsets = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        heights = np.array([a.shape[0] for a in images], np.int32)
        widths = np.array([a.shape[1] for a in images], np.int32)
        out = np.empty((n, self.embed_dim), np.float32)
        with self._stage_lock:
            buf = self._staging(int(offsets[-1]))
            self._fill(n, int(offsets[-1]),
                       lambda i: np.copyto(buf[offsets[i]:offsets[i + 1]].reshape(images[i].shape), images[i]))
            ptrs = (C.c_void_p * n)(*[self._stage_ptr.value + int(o) for o in offsets[:-1]])
            N.check(self._lib.b200_model_encode_images_u8_ragged(self._handle(), ptrs, _ptr(heights), _ptr(widths), n,
                                                                 1 if normalize else 0, _ptr(out)))
        return out

    def encode_images_u8(self, hwc: np.ndarray, normalize: bool = True) -> np.ndarray:
        a = _as(hwc, np.uint8)
        if a.ndim != 4 or a.shape[3] != 3:
            raise ValueError(f"expected uint8 [n, H, W, 3], got {a.shape}")
        out = np.empty((a.shape[0], self.embed_dim), np.float32)
        N.check(self._lib.b200_model_encode_images_u8(self._handle(), _ptr(a), a.shape[0], a.shape[1], a.shape[2],
                                                      1 if normalize else 0, _ptr(out)))
        return out

    def encode_images_f32(self, chw, normalize: bool = True) -> np.ndarray:
        a = _to_numpy_f32(chw)
        if a.ndim != 4 or a.shape[1] != 3 or a.shape[2] != self.image_size or a.shape[3] != self.image_size:
            raise ValueError(f"expected fp32 [n, 3, {self.image_size}, {self.image_size}], got {a.shape}")
        out = np.empty((a.shape[0], self.embed_dim), np.float32)
        N.check(self._lib.b200_model_encode_images_f32(self._handle(), _ptr(a), a.shape[0], 1 if normalize else 0,
                                                       _ptr(out)))
        return out

    def encode_tokens(self, ids, attn_mask=None, normalize: bool = True) -> np.ndarray:
        i = _as(ids.cpu().numpy() if hasattr(ids, "cpu") else ids, np.int32)
        if i.ndim != 2:
            raise ValueError(f"expected int [n, seq] token ids, got {i.shape}")
        mk = None
        if attn_mask is not None:
            mk = _as(attn_mask.cpu().numpy() if hasattr(attn_mask, "cpu") else attn_mask, np.int32)
            if mk.shape != i.shape:
                raise ValueError("attention mask shape must match ids")
        out = np.empty((i.shape[0], self.embed_dim), np.float32)
        N.check(self._lib.b200_model_encode_tokens(self._handle(), _ptr(i), _ptr(mk), i.shape[0], i.shape[1],
                                                   1 if normalize else 0, _ptr(out)))
        return out

    def classify_tokens(self, ids, attn_mask=None, type_ids=None, sigmoid: bool = True) -> np.ndarray:
        """A cross-encoder's scores (num_labels in the config) of sentence pairs: ids, attn_mask and type_ids int
        [n, seq] (None: all ones / all zeros) -> fp32 [n, num_labels], the logits through the sigmoid if sigmoid."""
        i = _as(ids.cpu().numpy() if hasattr(ids, "cpu") else ids, np.int32)
        if i.ndim != 2:
            raise ValueError(f"expected int [n, seq] token ids, got {i.shape}")
        extra = []
        for a in (attn_mask, type_ids):
            a = None if a is None else _as(a.cpu().numpy() if hasattr(a, "cpu") else a, np.int32)
            if a is not None and a.shape != i.shape:
                raise ValueError("attention mask and token-type ids must have the shape of the ids")
            extra.append(a)
        out = np.empty((i.shape[0], self.embed_dim), np.float32)
        N.check(self._lib.b200_model_classify_tokens(self._handle(), _ptr(i), _ptr(extra[0]), _ptr(extra[1]), i.shape[0],
                                                     i.shape[1], 1 if sigmoid else 0, _ptr(out)))
        return out

    def detect_images_u8(self, hwc, query_ids) -> Tuple[np.ndarray, np.ndarray]:
        """OWL-ViT detection (owl_detect in the config): uint8 [n, H, W, 3] images, squashed to image_size on the GPU,
        against one query's int ids [seq] (seq <= text ctx) -> (logits fp32 [n, G^2], boxes fp32 [n, G^2, 4] as
        (cx, cy, w, h) in [0, 1]), what OwlViTForObjectDetection returns as logits[..., 0] and pred_boxes."""
        a = _as(hwc, np.uint8)
        if a.ndim != 4 or a.shape[3] != 3:
            raise ValueError(f"expected uint8 [n, H, W, 3], got {a.shape}")
        q = _as(query_ids.cpu().numpy() if hasattr(query_ids, "cpu") else query_ids, np.int32).reshape(-1)
        P = self.grid * self.grid
        logits = np.empty((a.shape[0], P), np.float32)
        boxes = np.empty((a.shape[0], P, 4), np.float32)
        N.check(self._lib.b200_model_detect_images_u8(self._handle(), _ptr(a), a.shape[0], a.shape[1], a.shape[2],
                                                      _ptr(q), q.size, _ptr(logits), _ptr(boxes)))
        return logits, boxes

    def encode_videos_u8(self, thwc, normalize: bool = True) -> np.ndarray:
        """LanguageBind videos (video_frames in the config): uint8 RGB [n, T, H, W, 3] with T the model's frames,
        transformed on the GPU (short side to image_size, bilinear; centre crop; Normalize) -> fp32 [n, embed_dim]."""
        a = _as(thwc, np.uint8)
        if a.ndim != 5 or a.shape[4] != 3:
            raise ValueError(f"expected uint8 [n, T, H, W, 3], got {a.shape}")
        out = np.empty((a.shape[0], self.embed_dim), np.float32)
        N.check(self._lib.b200_model_encode_videos_u8(self._handle(), _ptr(a), a.shape[0], a.shape[1], a.shape[2],
                                                      a.shape[3], 1 if normalize else 0, _ptr(out)))
        return out

    def encode_videos_u8_device(self, d_ptr: int, n: int, t: int, h: int, w: int, d_out_ptr: int,
                                normalize: bool = True, sync: bool = True) -> None:
        N.check(self._lib.b200_model_encode_videos_u8_device(self._handle(), C.c_void_p(d_ptr), n, t, h, w,
                                                             1 if normalize else 0, C.c_void_p(d_out_ptr),
                                                             1 if sync else 0))

    def classify_tokens_device(self, d_ids_ptr: int, d_mask_ptr: Optional[int], d_types_ptr: Optional[int], n: int,
                               seq: int, d_out_ptr: int, sigmoid: bool = True, sync: bool = True) -> None:
        N.check(self._lib.b200_model_classify_tokens_device(self._handle(), C.c_void_p(d_ids_ptr),
                                                            C.c_void_p(d_mask_ptr) if d_mask_ptr else None,
                                                            C.c_void_p(d_types_ptr) if d_types_ptr else None, n, seq,
                                                            1 if sigmoid else 0, C.c_void_p(d_out_ptr),
                                                            1 if sync else 0))

    def encode_images_u8_device(self, d_ptr: int, n: int, h: int, w: int, d_out_ptr: int, normalize: bool = True,
                                sync: bool = True) -> None:
        N.check(self._lib.b200_model_encode_images_u8_device(self._handle(), C.c_void_p(d_ptr), n, h, w,
                                                             1 if normalize else 0, C.c_void_p(d_out_ptr),
                                                             1 if sync else 0))

    def encode_images_u8_ragged_device(self, ptrs: Sequence[int], heights: Sequence[int], widths: Sequence[int],
                                       d_out_ptr: int, normalize: bool = True, sync: bool = True) -> None:
        """Device-resident uint8 HWC images of any sizes: image i at device pointer ptrs[i], heights[i] x widths[i];
        d_out_ptr: fp32 device [n, embed_dim]."""
        n = len(ptrs)
        if len(heights) != n or len(widths) != n:
            raise ValueError(f"{n} pointers, {len(heights)} heights and {len(widths)} widths")
        p = (C.c_void_p * max(n, 1))(*[int(x) for x in ptrs])
        N.check(self._lib.b200_model_encode_images_u8_ragged_device(self._handle(), p, _ptr(_as(heights, np.int32)),
                                                                    _ptr(_as(widths, np.int32)), n,
                                                                    1 if normalize else 0, C.c_void_p(d_out_ptr),
                                                                    1 if sync else 0))

    def encode_tokens_device(self, d_ids_ptr: int, d_mask_ptr: Optional[int], n: int, seq: int, d_out_ptr: int,
                             normalize: bool = True, sync: bool = True) -> None:
        N.check(self._lib.b200_model_encode_tokens_device(self._handle(), C.c_void_p(d_ids_ptr),
                                                          C.c_void_p(d_mask_ptr) if d_mask_ptr else None, n, seq,
                                                          1 if normalize else 0, C.c_void_p(d_out_ptr),
                                                          1 if sync else 0))

    def set_stream(self, cuda_stream: Optional[int]) -> None:
        """cuda_stream: a cudaStream_t handle (0 = legacy default stream); None restores the private stream."""
        N.check(self._lib.b200_model_set_stream(self._handle(), C.c_void_p(cuda_stream or 0),
                                                0 if cuda_stream is None else 1))

    def set_profiling(self, on: bool) -> None:
        N.check(self._lib.b200_model_set_profiling(self._handle(), 1 if on else 0))

    def profile(self) -> dict:
        g, gn, a, an = C.c_float(0), C.c_int(0), C.c_float(0), C.c_int(0)
        N.check(self._lib.b200_model_profile(self._handle(), C.byref(g), C.byref(gn), C.byref(a), C.byref(an)))
        return {"gemm_ms": g.value, "gemm_launches": gn.value, "attention_ms": a.value, "attention_launches": an.value}

    def last_timing(self) -> Tuple[float, int]:
        ms, n = C.c_float(0), C.c_int(0)
        N.check(self._lib.b200_model_last_timing(self._handle(), C.byref(ms), C.byref(n)))
        return ms.value, n.value


# ---------------------------------------------------------------------------------------------------------
# Kernel-level diagnostics (b200_debug_*)
# ---------------------------------------------------------------------------------------------------------
class _Staging:
    """The device side of one b200_debug_* call: host arrays as torch tensors on cuda:{device}, and that device's
    current stream, which the hook runs on and synchronises.  The library looks for the device before torch touches
    CUDA, so without one the call fails with ERR_NO_DEVICE, as every compute entry point does."""

    def __init__(self, device: int):
        if not 0 <= device < N.device_count():
            raise N.NativeError(N.ERR_NO_DEVICE, f"CUDA device {device} not available (marqo_b200 has no CPU fallback)")
        import torch
        self.torch, self.device = torch, device
        self.dev = torch.device("cuda", device)
        self.stream = torch.cuda.current_stream(self.dev).cuda_stream

    def up(self, a, dtype: str = "float32"):
        """a (None stays None) on the device as `dtype` (a torch dtype name); "bfloat16" rounds fp32 values to nearest
        even, as __float2bfloat16_rn does."""
        if a is None:
            return None
        t = self.torch.from_numpy(_as(a, np.float32 if dtype == "bfloat16" else dtype)).to(self.dev)
        return t.to(getattr(self.torch, dtype))

    def empty(self, shape, dtype: str = "float32"):
        return self.torch.empty(shape, dtype=getattr(self.torch, dtype), device=self.dev)


def _dptr(t):
    return None if t is None else t.data_ptr()


def _host(t) -> np.ndarray:
    """A device tensor as a host array, bf16 widened to fp32."""
    return (t.float() if t.is_floating_point() else t).cpu().numpy()


def _gemm(d: _Staging, a, w, bias, residual, out, act: int = 0, sms: int = 0) -> int:
    """b200_debug_gemm: out[:M, :N] = act(a w^T + bias) (+ residual) for bf16 a [M, >= K], w [N, K] and out fp32 or
    bf16 [>= M, >= N]; residual may be out itself.  Returns the kernel that ran."""
    kernel = C.c_int(-1)
    N.check(N.load().b200_debug_gemm(d.device, _dptr(a), a.stride(0), _dptr(w), _dptr(bias), _dptr(residual),
                                     0 if residual is None else residual.stride(0), _dptr(out), out.stride(0),
                                     int(out.dtype == d.torch.bfloat16), act, a.shape[0], w.shape[0], w.shape[1], sms,
                                     C.byref(kernel), d.stream))
    return kernel.value


def debug_gemm(A, W, bias=None, residual=None, act: int = 0, out_bf16: bool = False, device: int = 0) -> np.ndarray:
    d = _Staging(device)
    a, w, b, r = d.up(A, "bfloat16"), d.up(W, "bfloat16"), d.up(bias), d.up(residual)
    out = d.empty((a.shape[0], w.shape[0]), "bfloat16" if out_bf16 else "float32")
    _gemm(d, a, w, b, r, out, act)
    return _host(out)


def debug_gemm_into(A, W, io, bias=None, act: int = 0, out_bf16: bool = False, residual_in_place: bool = False,
                    sms: Optional[int] = None, return_kernel: bool = False, device: int = 0):
    """GEMM into a copy of io (fp32 [rows >= M, cols >= N], bf16 on the device when out_bf16): rows [0, M) x columns
    [0, N) become act(A W^T + bias), plus their old values when residual_in_place (residual == out); the rest of the
    buffer is returned as the kernel left it.  The kernel is chosen by the library's rule for an SM count of sms (None:
    the device's own).  Returns the buffer, or with return_kernel (the buffer, the kernel that ran:
    _native.GEMM_128x128 or _native.GEMM_PERSISTENT)."""
    io = _as(io, np.float32)
    if io.ndim != 2 or io.shape[0] < len(A) or io.shape[1] < len(W):
        raise ValueError(f"io {io.shape} does not hold the [{len(A)}, {len(W)}] product")
    d = _Staging(device)
    a, w, b = d.up(A, "bfloat16"), d.up(W, "bfloat16"), d.up(bias)
    out = d.up(io, "bfloat16" if out_bf16 else "float32")
    kernel = _gemm(d, a, w, b, out if residual_in_place else None, out, act, sms or 0)
    return (_host(out), kernel) if return_kernel else _host(out)


def debug_scan_kernel(store: RowStore, force_streamed: Optional[bool] = None) -> int:
    """The scan kernel `store`'s last search ran (_native.SCAN_RESIDENT_Q or SCAN_STREAMED_Q; -1 before any search).
    force_streamed True makes later searches use the streamed-query kernel at any dim, False restores the library's
    rule, None leaves the setting as it is."""
    last = C.c_int(-1)
    force = -1 if force_streamed is None else int(bool(force_streamed))
    N.check(N.load().b200_debug_index_scan_kernel(store._handle(), force, C.byref(last)))
    return last.value


def debug_last_scan(store: RowStore) -> dict:
    """What `store`'s last search left on the device for its last query group (at most 64 queries):
    {"nq", "grid", "eps" fp32 [nq] (bound on |approximate - exact| scan key), "queries" fp32 [nq, dim] (the fp16 query
    block as scanned), "list_score" fp32 / "list_row" / "list_doc" int32 [grid, nq, _native.SCAN_LIST_LEN] (each scan
    CTA's best approximate keys per query)}.  nq = grid = 0 before any search."""
    lib, h = N.load(), store._handle()
    nq, grid = C.c_int(0), C.c_int(0)
    N.check(lib.b200_debug_index_last_scan(h, C.byref(nq), C.byref(grid), None, None, None, None, None))
    n, g = nq.value, grid.value
    eps = np.empty(n, np.float32)
    queries = np.empty((n, store.dim), np.float32)
    score = np.empty((g, n, N.SCAN_LIST_LEN), np.float32)
    row = np.empty((g, n, N.SCAN_LIST_LEN), np.int32)
    doc = np.empty((g, n, N.SCAN_LIST_LEN), np.int32)
    N.check(lib.b200_debug_index_last_scan(h, C.byref(nq), C.byref(grid), _ptr(eps), _ptr(queries), _ptr(score),
                                           _ptr(row), _ptr(doc)))
    if (nq.value, grid.value) != (n, g):
        raise RuntimeError("the store was searched between the two reads of its last scan")
    return {"nq": n, "grid": g, "eps": eps, "queries": queries, "list_score": score, "list_row": row, "list_doc": doc}


def debug_gemm_ln(A, W, bias, residual, gamma, beta, eps: float, in_place: bool = False, repeats: int = 1,
                  device: int = 0):
    """Residual GEMM followed by the LayerNorm launch, as the encoder layers run them, `repeats` times on the same
    buffers -> (x fp32 [M, N], LayerNorm(x) rounded to bf16 [M, N]).  in_place: the normalised fp32 rows also replace x
    (BERT's post-LN)."""
    if repeats < 1:
        raise ValueError(f"repeats must be positive, got {repeats}")
    d = _Staging(device)
    a, w, b, r = d.up(A, "bfloat16"), d.up(W, "bfloat16"), d.up(bias), d.up(residual)
    g, be = d.up(gamma), d.up(beta)
    M, Nn = a.shape[0], w.shape[0]
    x, ln = d.empty((M, Nn)), d.empty((M, Nn), "bfloat16")
    for _ in range(repeats):
        _gemm(d, a, w, b, r, x)
        N.check(N.load().b200_debug_layernorm(device, _dptr(x), Nn, _dptr(g), _dptr(be), float(eps), M, Nn,
                                              _dptr(x) if in_place else None, _dptr(ln), d.stream))
    return _host(x), _host(ln)


def debug_patch_embed(images_u8, patch: int, conv_w, mean, std, io, pos=None, cls=None, bias=None,
                      device: int = 0) -> np.ndarray:
    """The patch embedding of uint8 HWC images [n, S, S, 3] (G patches each) by the fused gather GEMM, into a copy of io
    (fp32 [rows >= M, cols >= N], N = len(conv_w)), in one of the forms the image forwards run
    (b200_debug_patch_embed):

      - pos given (fp32 [T, N]), the ViT form: rows [0, M = n T) become the token rows fed to ln_pre, T = G + 1 with a
        class row (cls fp32 [N]: cls + pos[0], then conv1(patch i) + pos[1 + i]), T = G without one (SigLIP:
        conv1(patch i) + pos[i]); io must have exactly N columns;
      - pos None, the ConvNeXt stem form: rows [0, M = n G) x columns [0, N) become conv1(patch i) + bias (None: no
        bias); cls must be None.

    Returns the whole buffer, the rest of it as the kernels left it."""
    img = _as(images_u8, np.uint8)
    n, S = img.shape[0], img.shape[1]
    w = _as(conv_w, np.float32).reshape(len(conv_w), -1)
    Nn = w.shape[0]
    T = (S // patch) ** 2 + (cls is not None)
    io = _as(io, np.float32)
    if io.ndim != 2 or io.shape[0] < n * T or io.shape[1] < Nn:
        raise ValueError(f"io {io.shape} does not hold the [{n * T}, {Nn}] token rows")
    if pos is not None and np.shape(pos) != (T, Nn):
        raise ValueError(f"pos {np.shape(pos)} is not [{T}, {Nn}]")
    m3, s3 = _as(mean, np.float32), _as(std, np.float32)
    d = _Staging(device)
    di, dw, out = d.up(img, "uint8"), d.up(w), d.up(io)
    dc, dp, db = d.up(cls), d.up(pos), d.up(bias)
    N.check(N.load().b200_debug_patch_embed(device, _dptr(di), n, S, patch, _dptr(dw), Nn, _ptr(m3), _ptr(s3),
                                            _dptr(dc), _dptr(dp), _dptr(db), _dptr(out), io.shape[1], d.stream))
    return _host(out)


def layer_cols(enc: Encoder, tower: str) -> Tuple[int, int, int]:
    """(width, aw, fc1) of a transformer tower's layer buffers, as the library lays them out (b200_debug_layer_cols):
    aw the attention width with every head zero-padded to the attention kernel's head dim, fc1 the columns fc1
    writes."""
    out = np.zeros(3, np.int32)
    N.check(enc._lib.b200_debug_layer_cols(enc._handle(), 0 if tower == "vision" else 1, _ptr(out)))
    return int(out[0]), int(out[1]), int(out[2])


def debug_layers(enc: Encoder, tower: str, first: int, count: int, x_in, S: int, kv_len=None) -> dict:
    """Layers [first, first + count) of enc's "vision" or "text" tower through the encoder's own layer runner, from
    the residual rows x_in fp32 [B * S, width] (a torch tensor on the encoder's device, or a host array), with key
    lengths kv_len [B] (each in 0..S) for the key-length towers (None: S each).  Returns what the last layer left, as
    device tensors: {"x": fp32 [B * S, width], "h": bf16 [B * S, width] the last LayerNorm output (pre-LN: fc1's
    input), "qkv": bf16 [B * S, 3 aw] after any rotary embedding, "o": bf16 [B * S, aw], "u": bf16 [B * S, fc1] after
    the activation or gate} (layer_cols gives aw and fc1)."""
    w, aw, fc1 = layer_cols(enc, tower)
    d = _Staging(enc.device)
    x = x_in.to(device=d.dev, dtype=d.torch.float32).contiguous() if hasattr(x_in, "to") else d.up(x_in)
    if x.dim() != 2 or x.shape[1] != w or S < 1 or x.shape[0] % S != 0:
        raise ValueError(f"expected x_in [B * {S}, {w}], got {tuple(x.shape)}")
    M = x.shape[0]
    kl = None if kv_len is None else d.up(kv_len, "int32")
    out = {"x": d.empty((M, w)), "h": d.empty((M, w), "bfloat16"), "qkv": d.empty((M, 3 * aw), "bfloat16"),
           "o": d.empty((M, aw), "bfloat16"), "u": d.empty((M, fc1), "bfloat16")}
    N.check(enc._lib.b200_debug_layers(enc._handle(), 0 if tower == "vision" else 1, first, count, _dptr(x), M // S,
                                       S, _dptr(kl), _dptr(out["x"]), _dptr(out["h"]), _dptr(out["qkv"]),
                                       _dptr(out["o"]), _dptr(out["u"]), d.stream))
    return out


def debug_attention(qkv, B: int, S: int, W: int, H: int, mask: int = 0, kv_len=None, device: int = 0,
                    rel_bias=None) -> np.ndarray:
    """softmax(q k^T / sqrt(hd) + mask) v over packed qkv.  rel_bias: MPNet's relative-position bias, fp32
    [H, 2 * smax - 1], adds rel_bias[h, j - i + smax - 1] to the logit of query i and key j (key-length mask only,
    head_dim 64, S <= smax)."""
    rb, smax = None, 0
    if rel_bias is not None:
        rb = _as(rel_bias, np.float32)
        if mask != 2 or kv_len is None:
            raise ValueError("the relative bias runs with the key-length mask (mask=2, kv_len)")
        if rb.ndim != 2 or rb.shape[0] != H or rb.shape[1] % 2 != 1:
            raise ValueError(f"expected rel_bias [{H}, 2 * smax - 1], got {rb.shape}")
        smax = (rb.shape[1] + 1) // 2
    d = _Staging(device)
    q, kl = d.up(qkv, "bfloat16"), d.up(kv_len, "int32")
    out = d.empty((B * S, W), "bfloat16")
    N.check(N.load().b200_debug_attention(device, _dptr(q), B, S, W, H, mask, _dptr(kl), _ptr(rb), smax, _dptr(out),
                                          d.stream))
    return _host(out)


def debug_attention_time(B: int, S: int, W: int, H: int, mask: int = 0, rel_bias: bool = False, iters: int = 20,
                         device: int = 0) -> float:
    """Mean device time (ms) of the attention launch on generated data, every key kept; rel_bias adds a generated
    relative-position bias (with mask=2)."""
    ms = C.c_float(0)
    N.check(N.load().b200_debug_attention_time(device, B, S, W, H, mask, int(rel_bias), iters, C.byref(ms)))
    return ms.value


def relative_position_buckets(max_len: int, num_buckets: int = 32, max_distance: int = 128) -> np.ndarray:
    """The bucket of every key - query distance d, |d| < max_len, as the MPNet runtime builds its bias table:
    out[d + max_len - 1]."""
    out = np.empty(2 * max_len - 1, np.int32)
    N.check(N.load().b200_debug_relative_position_buckets(num_buckets, max_distance, max_len, _ptr(out)))
    return out


def debug_layernorm(x, gamma, beta, eps: float, rows: Optional[int] = None, in_stride: int = 0, outputs: str = "f32",
                    in_place: bool = False, device: int = 0):
    """LayerNorm of `rows` rows of width w = len(gamma), row r read at x.flat[r * in_stride] (in_stride 0: w; rows None:
    x.size // in_stride).  outputs "f32" returns the fp32 output [rows, w], "bf16" the bf16 output (as fp32), "both"
    the pair (fp32, bf16) of one launch.  in_place writes the fp32 output over x on the device, as ln_pre and BERT's
    post-LN do."""
    if outputs not in ("f32", "bf16", "both"):
        raise ValueError(f"outputs must be 'f32', 'bf16' or 'both', got {outputs!r}")
    xa, g, b = _as(x, np.float32).reshape(-1), _as(gamma, np.float32), _as(beta, np.float32)
    w = g.size
    stride = in_stride or w
    if rows is None:
        rows = xa.size // stride
    if b.size != w or rows < 1 or stride < w or xa.size < (rows - 1) * stride + w:
        raise ValueError(f"x of {xa.size} floats does not hold {rows} rows of {w} at stride {stride}")
    if in_place and (outputs == "bf16" or stride != w):
        raise ValueError("in place needs the fp32 output and compact rows")
    d = _Staging(device)
    dx, dg, db = d.up(xa), d.up(g), d.up(b)
    f = h = None
    if outputs != "bf16":
        f = dx[:rows * w].view(rows, w) if in_place else d.empty((rows, w))
    if outputs != "f32":
        h = d.empty((rows, w), "bfloat16")
    N.check(N.load().b200_debug_layernorm(device, _dptr(dx), in_stride, _dptr(dg), _dptr(db), eps, rows, w, _dptr(f),
                                          _dptr(h), d.stream))
    f, h = (None if t is None else _host(t) for t in (f, h))
    return (f, h) if outputs == "both" else (f if h is None else h)


def debug_clip_text_embed(ids, tok, pos, device: int = 0, cls=None):
    """CLIP / SigLIP text embedding of ids int32 [n, S]: (x fp32 [n*S, w] = tok[ids] + pos[s], eot int32 [n]).
    cls fp32 [w] (CoCa): S + 1 rows per sequence, the last one cls + pos[S], and eot = S."""
    ia, t, p = _as(ids, np.int32), _as(tok, np.float32), _as(pos, np.float32)
    n, S = ia.shape
    vocab, w = t.shape
    rows = S + (cls is not None)
    if p.shape != (rows, w):
        raise ValueError(f"expected pos [{rows}, {w}], got {p.shape}")
    d = _Staging(device)
    di, dt, dp = d.up(ia, "int32"), d.up(t), d.up(p)
    x, eot = d.empty((n * rows, w)), d.empty(n, "int32")
    if cls is None:
        N.check(N.load().b200_debug_clip_text_embed(device, _dptr(di), _dptr(dt), _dptr(dp), n, S, w, vocab, _dptr(x),
                                                    _dptr(eot), d.stream))
    else:
        dc = d.up(_as(cls, np.float32))
        N.check(N.load().b200_debug_clip_text_embed_cls(device, _dptr(di), _dptr(dt), _dptr(dp), _dptr(dc), n, rows, w,
                                                        vocab, _dptr(x), _dptr(eot), d.stream))
    return _host(x), _host(eot)


def debug_embed_ln(ids, mask, word, pos, type0, gamma, beta, eps: float, pad: Optional[int] = None, device: int = 0,
                   type_ids=None):
    """BERT (pad None; pos None for GTE, which has no position table) or RoBERTa (pad = the pad id; type0 None for
    MPNet) embedding + LayerNorm of ids int32 [n, S] with an optional mask [n, S] -> (x fp32 [n*S, w], its bf16 copy as
    fp32, kv_len int32 [n]).  type_ids (BERT with positions: a sentence pair's int32 [n, S]): type0 is the whole
    token-type table [rows, w] and each token adds its own row."""
    ia, wd = _as(ids, np.int32), _as(word, np.float32)
    p = None if pos is None else _as(pos, np.float32)
    n, S = ia.shape
    vocab, w = wd.shape
    m = None if mask is None else _as(mask, np.int32)
    t = None if type0 is None else _as(type0, np.float32)
    ti = None if type_ids is None else _as(type_ids, np.int32)
    g, b = _as(gamma, np.float32), _as(beta, np.float32)
    if m is not None and m.shape != ia.shape:
        raise ValueError(f"expected mask {ia.shape}, got {m.shape}")
    if ti is not None and (ti.shape != ia.shape or t is None or t.ndim != 2 or t.shape[1] != w):
        raise ValueError(f"type_ids must be {ia.shape} with a token-type table [rows, {w}]")
    type_rows = 0 if ti is None else t.shape[0]
    need = S if pad is None else pad + S + 1
    if p is not None and (p.ndim != 2 or p.shape[1] != w or p.shape[0] < need):
        raise ValueError(f"expected pos [>= {need}, {w}], got {p.shape}")
    if (t is not None and ti is None and t.size != w) or g.size != w or b.size != w:
        raise ValueError(f"type0, gamma and beta must have {w} values")
    d = _Staging(device)
    di, dm, dwd, dp, dt = d.up(ia, "int32"), d.up(m, "int32"), d.up(wd), d.up(p), d.up(t)
    dti = d.up(ti, "int32")
    dg, db = d.up(g), d.up(b)
    x, h, kv_len = d.empty((n * S, w)), d.empty((n * S, w), "bfloat16"), d.empty(n, "int32")
    N.check(N.load().b200_debug_embed_ln(device, _dptr(di), _dptr(dm), _dptr(dwd), _dptr(dp),
                                         0 if p is None else p.shape[0], _dptr(dt),
                                         _dptr(dg), _dptr(db), eps, n, S, w, vocab, -1 if pad is None else pad, _dptr(x),
                                         _dptr(h), _dptr(kv_len), _dptr(dti), type_rows, d.stream))
    return _host(x), _host(h), _host(kv_len)


def debug_clip_head(x, S: int, gamma, beta, eps: float, proj, row_in_seq=None, normalize: bool = True,
                    device: int = 0) -> np.ndarray:
    """CLIP head over token rows x fp32 [n*S, w]: LN(x[b*S + row_in_seq[b]]) @ proj [w, E] (row_in_seq None: row 0),
    L2-normalised if normalize -> fp32 [n, E]."""
    xa, pj = _as(x, np.float32), _as(proj, np.float32)
    w, E = pj.shape
    if xa.ndim != 2 or xa.shape[1] != w or xa.shape[0] % S != 0:
        raise ValueError(f"expected x [n * {S}, {w}], got {xa.shape}")
    n = xa.shape[0] // S
    r = None if row_in_seq is None else _as(row_in_seq, np.int32)
    if r is not None and (r.shape != (n,) or r.min() < 0 or r.max() >= S):
        raise ValueError(f"row_in_seq must be [{n}] rows in [0, {S})")
    g, b = _as(gamma, np.float32), _as(beta, np.float32)
    d = _Staging(device)
    dx, dr, dg, db, dp = d.up(xa), d.up(r, "int32"), d.up(g), d.up(b), d.up(pj)
    out = d.empty((n, E))
    N.check(N.load().b200_debug_clip_head(device, _dptr(dx), S, _dptr(dr), _dptr(dg), _dptr(db), eps, _dptr(dp), n, w,
                                          E, int(normalize), _dptr(out), d.stream))
    return _host(out)


def debug_bert_head(x, S: int, kv_len, pool: int = N.POOL_MEAN, normalize: bool = True, device: int = 0) -> np.ndarray:
    """BERT head over x fp32 [n*S, w]: mean of the first kv_len[b] rows (POOL_MEAN) or row 0 (POOL_CLS), F.normalize'd
    if normalize -> fp32 [n, w]."""
    xa = _as(x, np.float32)
    if xa.ndim != 2 or xa.shape[0] % S != 0:
        raise ValueError(f"expected x [n * {S}, w], got {xa.shape}")
    n, w = xa.shape[0] // S, xa.shape[1]
    kl = _as(kv_len, np.int32)
    if kl.shape != (n,):
        raise ValueError(f"expected kv_len [{n}], got {kl.shape}")
    d = _Staging(device)
    dx, dkl = d.up(xa), d.up(kl, "int32")
    out = d.empty((n, w))
    N.check(N.load().b200_debug_bert_head(device, _dptr(dx), _dptr(dkl), n, S, w, pool, int(normalize), _dptr(out),
                                          d.stream))
    return _host(out)


def debug_text_head(x, S: int, kv_len, proj, bias=None, normalize: bool = True, device: int = 0) -> np.ndarray:
    """M-CLIP's text head over x fp32 [n*S, w]: the mean of the first kv_len[b] rows @ proj [w, E] + bias [E] (None:
    none), divided by its L2 norm if normalize -> fp32 [n, E]."""
    xa, pj = _as(x, np.float32), _as(proj, np.float32)
    w, E = pj.shape
    if xa.ndim != 2 or xa.shape[1] != w or xa.shape[0] % S != 0:
        raise ValueError(f"expected x [n * {S}, {w}], got {xa.shape}")
    n = xa.shape[0] // S
    kl = _as(kv_len, np.int32)
    if kl.shape != (n,):
        raise ValueError(f"expected kv_len [{n}], got {kl.shape}")
    b = None if bias is None else _as(bias, np.float32)
    d = _Staging(device)
    dx, dkl, dp, dbias = d.up(xa), d.up(kl, "int32"), d.up(pj), d.up(b)
    out = d.empty((n, E))
    N.check(N.load().b200_debug_text_head(device, _dptr(dx), _dptr(dkl), n, S, w, _dptr(dp), _dptr(dbias), E,
                                          int(normalize), _dptr(out), d.stream))
    return _host(out)


def debug_cls_head(x, S: int, pool_w, pool_b, cls_w, cls_b, sigmoid: bool = False, device: int = 0) -> np.ndarray:
    """BertForSequenceClassification's head over x fp32 [n*S, w]: tanh(pool_w [w, w] . x[b*S] + pool_b) through the
    classifier cls_w [L, w], cls_b [L], then the sigmoid if sigmoid -> fp32 [n, L]."""
    xa, pw, pb, cw, cb = (_as(a, np.float32) for a in (x, pool_w, pool_b, cls_w, cls_b))
    w, L = pw.shape[0], cw.shape[0]
    if xa.ndim != 2 or xa.shape[1] != w or xa.shape[0] % S != 0:
        raise ValueError(f"expected x [n * {S}, {w}], got {xa.shape}")
    if pw.shape != (w, w) or pb.shape != (w,) or cw.shape != (L, w) or cb.shape != (L,):
        raise ValueError("expected pool_w [w, w], pool_b [w], cls_w [L, w], cls_b [L]")
    n = xa.shape[0] // S
    d = _Staging(device)
    dx, dpw, dpb, dcw, dcb = d.up(xa), d.up(pw), d.up(pb), d.up(cw), d.up(cb)
    out = d.empty((n, L))
    N.check(N.load().b200_debug_cls_head(device, _dptr(dx), n, S, w, _dptr(dpw), _dptr(dpb), _dptr(dcw), _dptr(dcb), L,
                                         int(sigmoid), _dptr(out), d.stream))
    return _host(out)


def debug_owl_merge_ln(x, N_rows: int, post_g, post_b, det_g, det_b, eps: float = 1e-5, device: int = 0) -> np.ndarray:
    """OWL-ViT's patch features over trunk rows x fp32 [n * N_rows, w] (class row first per image): LN_det(LN_post(patch)
    * LN_post(class)) -> fp32 [n * (N_rows - 1), w] (the kernel's bf16 values, widened)."""
    xa = _as(x, np.float32)
    w = xa.shape[1]
    n = xa.shape[0] // N_rows
    d = _Staging(device)
    dx, g1, b1, g2, b2 = (d.up(a) for a in (xa, post_g, post_b, det_g, det_b))
    out = d.empty((n * (N_rows - 1), w), "bfloat16")
    N.check(N.load().b200_debug_owl_merge_ln(device, _dptr(dx), n, N_rows, w, _dptr(g1), _dptr(b1), _dptr(g2), _dptr(b2),
                                             float(eps), _dptr(out), d.stream))
    return _host(out.float())


def debug_owl_class_logits(c, E: int, t, device: int = 0) -> np.ndarray:
    """OWL-ViT's class logits from class-head GEMM rows c fp32 [M, ldc] (dense0 | shift | scale | padding) and the
    query's text embedding t fp32 [E] -> fp32 [M]."""
    ca, ta = _as(c, np.float32), _as(t, np.float32)
    d = _Staging(device)
    dc, dt = d.up(ca), d.up(ta)
    out = d.empty((ca.shape[0],))
    N.check(N.load().b200_debug_owl_class_logits(device, _dptr(dc), ca.shape[1], ca.shape[0], int(E), _dptr(dt),
                                                 _dptr(out), d.stream))
    return _host(out)


def debug_owl_boxes(a, P: int, w2, b2, box_bias, device: int = 0) -> np.ndarray:
    """OWL-ViT's boxes from the box head's second GELU rows a [M, w] (rounded to bf16) -> fp32 [M, 4]."""
    aa = _as(a, np.float32)
    d = _Staging(device)
    da, dw, db, dbb = d.up(aa, "bfloat16"), d.up(w2), d.up(b2), d.up(box_bias)
    out = d.empty((aa.shape[0], 4))
    N.check(N.load().b200_debug_owl_boxes(device, _dptr(da), aa.shape[0], aa.shape[1], int(P), _dptr(dw), _dptr(db),
                                          _dptr(dbb), _dptr(out), d.stream))
    return _host(out)


def owl_box_bias(G: int) -> np.ndarray:
    """The engine's OWL-ViT box bias table of a G x G grid, fp32 [G^2, 4] (built on the host: no device needed)."""
    out = np.empty((G * G, 4), np.float32)
    N.check(N.load().b200_debug_owl_box_bias(int(G), _ptr(out)))
    return out


def debug_frame_mean_head(x, N_rows: int, T: int, gamma, beta, eps: float, proj, scale: float = 1.0,
                          row_in_seq=None, normalize: bool = True, device: int = 0) -> np.ndarray:
    """LanguageBind's heads over x fp32 [n * T * N_rows, w]: the mean over the T rows (b T + t) N_rows + r (r =
    row_in_seq[b], None: 0) of their LayerNorm, @ proj [w, E], v / |v| * scale, then / its norm if normalize."""
    d = _Staging(device)
    xa = _as(x, np.float32)
    pr = _as(proj, np.float32)
    w, E = xa.shape[1], pr.shape[1]
    n = xa.shape[0] // (T * N_rows)
    dx, dg, db, dp = d.up(xa), d.up(gamma), d.up(beta), d.up(pr)
    dr = d.up(row_in_seq, "int32")
    out = d.empty((n, E))
    N.check(N.load().b200_debug_frame_mean_head(device, _dptr(dx), N_rows, T, _dptr(dr), _dptr(dg), _dptr(db), eps,
                                                _dptr(dp), n, w, E, float(scale), 1 if normalize else 0, _dptr(out),
                                                d.stream))
    return _host(out)


def debug_temporal_embed_ln(x, temb, N_rows: int, T: int, gamma, beta, eps: float, device: int = 0):
    """LanguageBind's temporal step: (x + temb[(r / N_rows) % T] fp32 [rows, w], bf16 LN of it as fp32)."""
    d = _Staging(device)
    xa = _as(x, np.float32)
    rows, w = xa.shape
    dx, dt, dg, db = d.up(xa), d.up(temb), d.up(gamma), d.up(beta)
    h = d.empty((rows, w), "bfloat16")
    N.check(N.load().b200_debug_temporal_embed_ln(device, _dptr(dx), _dptr(dt), N_rows, T, _dptr(dg), _dptr(db), eps,
                                                  rows, w, _dptr(h), d.stream))
    return _host(dx), _host(h.float())


def debug_temporal_attention(qkv, n: int, T: int, N_rows: int, H: int, device: int = 0) -> np.ndarray:
    """Attention over the T frames of each (video, token) pair: qkv [n * T * N_rows, 3W] (rounded to bf16), heads of
    64 -> out [n * T * N_rows, W] (bf16 values as fp32)."""
    d = _Staging(device)
    q = d.up(qkv, "bfloat16")
    W = q.shape[1] // 3
    out = d.empty((q.shape[0], W), "bfloat16")
    N.check(N.load().b200_debug_temporal_attention(device, _dptr(q), n, T, N_rows, W, H, _dptr(out), d.stream))
    return _host(out.float())


def debug_temporal_attention_time(n: int, T: int, N_rows: int, W: int, H: int, iters: int = 50,
                                  device: int = 0) -> float:
    ms = C.c_float(0)
    N.check(N.load().b200_debug_temporal_attention_time(device, n, T, N_rows, W, H, iters, C.byref(ms)))
    return ms.value


def debug_video_resize_crop(frames, S: int, mean, std, device: int = 0) -> np.ndarray:
    """LanguageBind's video transform of uint8 RGB frames [f, h, w, 3] -> fp32 CHW [f, 3, S, S]."""
    d = _Staging(device)
    a = _as(frames, np.uint8)
    f, h, w, _ = a.shape
    da = d.up(a, "uint8")
    out = d.empty((f, 3, S, S))
    m3, s3 = np.asarray(mean, np.float32), np.asarray(std, np.float32)
    N.check(N.load().b200_debug_video_resize_crop(device, _dptr(da), f, h, w, S, _ptr(m3), _ptr(s3), _dptr(out),
                                                  d.stream))
    return _host(out)


def debug_l2_rows(src, normalize: bool = True, device: int = 0) -> np.ndarray:
    """src fp32 [n, E] -> each row divided by its L2 norm if normalize, else a copy."""
    a = _as(src, np.float32)
    if a.ndim != 2:
        raise ValueError(f"expected [n, E], got {a.shape}")
    d = _Staging(device)
    da, out = d.up(a), d.empty(a.shape)
    N.check(N.load().b200_debug_l2_rows(device, _dptr(da), a.shape[0], a.shape[1], int(normalize), _dptr(out),
                                        d.stream))
    return _host(out)


def debug_stem_im2col(images, mean=(0.0, 0.0, 0.0), std=(1.0, 1.0, 1.0), device: int = 0) -> np.ndarray:
    """ResNet stem im2col of uint8 HWC [n, S, S, 3] (normalised with mean / std) or already-normalised fp32 CHW
    [n, 3, S, S] -> fp32 [n * (S/2)^2, 64] (rounded to bf16), k = (3 ky + kx) * 3 + c."""
    u8 = images.dtype == np.uint8
    a = _as(images, np.uint8 if u8 else np.float32)
    n, S = a.shape[0], a.shape[1] if u8 else a.shape[2]
    if a.shape != ((n, S, S, 3) if u8 else (n, 3, S, S)) or S % 2 != 0:
        raise ValueError(f"expected [n, S, S, 3] uint8 or [n, 3, S, S] fp32 with S even, got {a.shape}")
    m3, s3 = _as(mean, np.float32), _as(std, np.float32)
    d = _Staging(device)
    da = d.up(a, "uint8" if u8 else "float32")
    out = d.empty((n * (S // 2) ** 2, 64), "bfloat16")
    N.check(N.load().b200_debug_stem_im2col(device, _dptr(da) if u8 else None, None if u8 else _dptr(da), n, S,
                                            _ptr(m3), _ptr(s3), _dptr(out), d.stream))
    return _host(out)


def debug_avgpool2(x, device: int = 0) -> np.ndarray:
    """AvgPool2d(2) over NHWC fp32 [n, H, W, C] (rounded to bf16) -> [n, H/2, W/2, C] (rounded to bf16)."""
    a = _as(x, np.float32)
    n, H, W, Cc = a.shape
    if H % 2 or W % 2 or Cc % 8:
        raise ValueError(f"H, W must be even and C a multiple of 8, got {a.shape}")
    d = _Staging(device)
    da, out = d.up(a, "bfloat16"), d.empty((n, H // 2, W // 2, Cc), "bfloat16")
    N.check(N.load().b200_debug_avgpool2(device, _dptr(da), n, H, W, Cc, _dptr(out), d.stream))
    return _host(out)


def debug_attnpool_tokens(x, pos, device: int = 0) -> np.ndarray:
    """ResNet attention-pool tokens: x fp32 [n, HW, C] (rounded to bf16), pos fp32 [HW + 1, C] -> [n, HW + 1, C]
    (rounded to bf16): row 0 = mean_s x_s + pos[0], row 1 + s = x_s + pos[1 + s]."""
    a, p = _as(x, np.float32), _as(pos, np.float32)
    n, HW, Cc = a.shape
    if p.shape != (HW + 1, Cc) or Cc % 8:
        raise ValueError(f"expected pos [{HW + 1}, {Cc}] and C a multiple of 8, got {p.shape}")
    d = _Staging(device)
    da, dp, out = d.up(a, "bfloat16"), d.up(p), d.empty((n, HW + 1, Cc), "bfloat16")
    N.check(N.load().b200_debug_attnpool_tokens(device, _dptr(da), _dptr(dp), n, HW, Cc, _dptr(out), d.stream))
    return _host(out)


def debug_im2col_f32(chw, patch: int, kpad: int, cls: int, device: int = 0) -> np.ndarray:
    """ViT im2col of fp32 CHW [n, 3, S, S] -> fp32 [n * ((S/p)^2 + cls), kpad] (rounded to bf16): the class rows
    (cls = 1) and the columns past 3 p^2 are zero."""
    a = _as(chw, np.float32)
    n, c, S, S2 = a.shape
    if c != 3 or S != S2 or S % patch or kpad % 8 or kpad < 3 * patch * patch or cls not in (0, 1):
        raise ValueError(f"bad im2col shape {a.shape}, patch {patch}, kpad {kpad}, cls {cls}")
    d = _Staging(device)
    da, out = d.up(a), d.empty((n * ((S // patch) ** 2 + cls), kpad), "bfloat16")
    N.check(N.load().b200_debug_im2col_f32(device, _dptr(da), n, S, patch, kpad, cls, _dptr(out), d.stream))
    return _host(out)


def debug_resize(hwc, S: int, device: int = 0) -> np.ndarray:
    a = _as(hwc, np.uint8)
    d = _Staging(device)
    da, out = d.up(a, "uint8"), d.empty((a.shape[0], S, S, 3), "uint8")
    N.check(N.load().b200_debug_resize(device, _dptr(da), a.shape[0], a.shape[1], a.shape[2], S, _dptr(out), d.stream))
    return _host(out)


def debug_resize_squash(hwc, S: int, device: int = 0) -> np.ndarray:
    """uint8 [n, h, w, 3] -> [n, S, S, 3] as PIL resize((S, S), BICUBIC) does (SigLIP's squash resize)."""
    a = _as(hwc, np.uint8)
    d = _Staging(device)
    da, out = d.up(a, "uint8"), d.empty((a.shape[0], S, S, 3), "uint8")
    N.check(N.load().b200_debug_resize_squash(device, _dptr(da), a.shape[0], a.shape[1], a.shape[2], S, _dptr(out),
                                              d.stream))
    return _host(out)


def debug_resize_ragged(images, S: int, squash: bool = False, device: int = 0) -> np.ndarray:
    """uint8 HWC images of any sizes -> uint8 [n, S, S, 3] in one ragged resize: the shortest side to S and the centre
    crop (as debug_resize), or with squash both sides to S (as debug_resize_squash)."""
    imgs = [_as(a, np.uint8) for a in images]
    d = _Staging(device)
    dev = [d.up(a, "uint8") for a in imgs]
    heights = np.array([a.shape[0] for a in imgs], np.int32)
    widths = np.array([a.shape[1] for a in imgs], np.int32)
    out = d.empty((len(imgs), S, S, 3), "uint8")
    ptrs = (C.c_void_p * max(len(imgs), 1))(*[t.data_ptr() for t in dev])
    N.check(N.load().b200_debug_resize_ragged(device, ptrs, _ptr(heights), _ptr(widths), len(imgs), S, int(squash),
                                              _dptr(out), d.stream))
    return _host(out)


def debug_map_attention(q, kv, B: int, S: int, H: int, device: int = 0) -> np.ndarray:
    """Single-query attention pooling: q fp32 [W] (SigLIP's one latent query, shared by every image) or [B, W] (one
    query per image, the ResNet attention pool), kv [B * S, 2W] (K then V columns, rounded to bf16) -> fp32 [B, W],
    softmax(q_h k_h^T / sqrt(D)) v_h per image and head of D = W / H columns, 64 or 96 (rounded to bf16)."""
    qa, kva = _as(q, np.float32), _as(kv, np.float32)
    W = qa.shape[-1]
    if qa.ndim not in (1, 2) or (qa.ndim == 2 and qa.shape[0] != B):
        raise ValueError(f"expected q [{W}] or [{B}, {W}], got {qa.shape}")
    if kva.shape != (B * S, 2 * W):
        raise ValueError(f"expected kv [{B * S}, {2 * W}], got {kva.shape}")
    d = _Staging(device)
    dq, dkv, out = d.up(qa), d.up(kva, "bfloat16"), d.empty((B, W), "bfloat16")
    N.check(N.load().b200_debug_map_attention(device, _dptr(dq), 0 if qa.ndim == 1 else W, _dptr(dkv), B, S, W, H,
                                              _dptr(out), d.stream))
    return _host(out)


def debug_conv2d(x, w, bias=None, residual=None, relu: bool = True, device: int = 0) -> np.ndarray:
    """One convolution of the ResNet CLIP image tower on the path the model runs it: x NHWC fp32 [n, H, W, cin], w
    [cout, cin, k, k] (torch layout), bias [cout] -> NHWC [n, Ho, Wo, cout] rounded to bf16: relu(conv + bias
    (+ residual)), or conv + bias without relu (1 x 1 and stem convs, no residual).  cin 3 is the stem conv (3 x 3, stride 2, padding 1);
    otherwise k 1 or 3 (stride 1, padding 1).  Operands are rounded to bf16 on the device."""
    xa, wa = _as(x, np.float32), _as(w, np.float32)
    n, H, W, cin = xa.shape
    cout, k = wa.shape[0], wa.shape[2]
    if wa.shape != (cout, cin, k, k):
        raise ValueError(f"expected w [cout, {cin}, k, k], got {wa.shape}")
    Ho, Wo = (H // 2, W // 2) if cin == 3 else (H, W)
    r = None if residual is None else _as(residual, np.float32)
    if r is not None and r.shape != (n, Ho, Wo, cout):
        raise ValueError(f"expected residual [{n}, {Ho}, {Wo}, {cout}], got {r.shape}")
    d = _Staging(device)
    # the stem reads fp32 CHW, as the fp32 image entry point receives it; the other convs a bf16 NHWC activation
    dx = d.up(xa).permute(0, 3, 1, 2).contiguous() if cin == 3 else d.up(xa, "bfloat16")
    db = d.up(np.zeros(cout) if bias is None else bias)
    dr, out = d.up(r, "bfloat16"), d.empty((n, Ho, Wo, cout), "bfloat16")
    N.check(N.load().b200_debug_conv2d(device, _dptr(dx), n, H, W, cin, _ptr(wa), cout, k, _dptr(db), _dptr(dr),
                                       int(relu), _dptr(out), d.stream))
    return _host(out)


def _ln_args(gamma, beta, C: int):
    g, b = _as(gamma, np.float32), _as(beta, np.float32)
    if g.shape != (C,) or b.shape != (C,):
        raise ValueError(f"expected gamma and beta [{C}], got {g.shape} and {b.shape}")
    return g, b


def debug_dwconv7_ln(x, w, bias, gamma, beta, eps: float, device: int = 0) -> np.ndarray:
    """ConvNeXt block head: x NHWC fp32 [n, H, W, C], w [C, 1, 7, 7] (conv_dw.weight), bias [C] -> fp32 [n * H * W, C]
    (rounded to bf16) = LayerNorm over C of the 7 x 7 depthwise conv (zero padding 3) plus bias."""
    xa, wa = _as(x, np.float32), _as(w, np.float32)
    n, H, W, Cc = xa.shape
    if wa.shape != (Cc, 1, 7, 7):
        raise ValueError(f"expected w [{Cc}, 1, 7, 7], got {wa.shape}")
    g, b = _ln_args(gamma, beta, Cc)
    d = _Staging(device)
    taps = np.ascontiguousarray(wa.reshape(Cc, 49).T)   # [49, C], as the model lays it out
    dx, dw, db, dg, dbeta = d.up(xa), d.up(taps), d.up(bias), d.up(g), d.up(b)
    out = d.empty((n * H * W, Cc), "bfloat16")
    N.check(N.load().b200_debug_dwconv7_ln(device, _dptr(dx), n, H, W, Cc, _dptr(dw), _dptr(db), _dptr(dg), _dptr(dbeta),
                                           float(eps), _dptr(out), d.stream))
    return _host(out)


def debug_ln_pixels(x, gamma, beta, eps: float, patchify: bool, device: int = 0) -> np.ndarray:
    """ConvNeXt per-pixel LayerNorm of x NHWC fp32 [n, H, W, C].  patchify False: fp32 [n * H * W, C] (the stem's norm,
    written in place over x on the device); True: [n * (H/2) * (W/2), 4C] rounded to bf16, the downsample conv's GEMM
    rows, pixel (y, x) at columns ((y % 2) * 2 + x % 2) * C + c of row (y/2, x/2)."""
    xa = _as(x, np.float32)
    n, H, W, Cc = xa.shape
    if patchify and (H % 2 or W % 2):
        raise ValueError(f"patchify needs an even H and W, got {xa.shape}")
    g, b = _ln_args(gamma, beta, Cc)
    d = _Staging(device)
    dx, dg, dbeta = d.up(xa), d.up(g), d.up(b)
    out = d.empty((n * H * W // 4, 4 * Cc), "bfloat16") if patchify else dx
    N.check(N.load().b200_debug_ln_pixels(device, _dptr(dx), n, H, W, Cc, _dptr(dg), _dptr(dbeta), float(eps),
                                          int(patchify), _dptr(out), d.stream))
    return _host(out).reshape(-1, 4 * Cc if patchify else Cc)


def debug_pool_ln(x, gamma, beta, eps: float, device: int = 0) -> np.ndarray:
    """ConvNeXt head input: x fp32 [n, HW, C] -> fp32 [n, C] (rounded to bf16) = LayerNorm over C of the mean over the
    HW pixels of each image."""
    xa = _as(x, np.float32)
    n, HW, Cc = xa.shape
    g, b = _ln_args(gamma, beta, Cc)
    d = _Staging(device)
    dx, dg, dbeta, out = d.up(xa), d.up(g), d.up(b), d.empty((n, Cc), "bfloat16")
    N.check(N.load().b200_debug_pool_ln(device, _dptr(dx), n, HW, Cc, _dptr(dg), _dptr(dbeta), float(eps), _dptr(out),
                                        d.stream))
    return _host(out)
