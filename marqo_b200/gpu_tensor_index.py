"""`VespaClient`-shaped adapter over the GPU row store (boundary B2, SURVEY §8b / a8 / a9 / f1).

Drop-in for `Config.vespa_client` (src/marqo/config.py:35) on the dense path: `feed_batch` / `query` / `get_batch` /
`delete_batch` keep the argument meaning and the response shapes of src/marqo/vespa/vespa_client.py:198-242,
:267-296, :405-440, :468-500 and src/marqo/vespa/models/{query_result,feed_response,get_document_response,
delete_document_response}.py.  Tensor queries (ranking == 'embedding_similarity', YQL made only of
`nearestNeighbor(...)` terms, optionally followed by the ` AND <filter>` text either index type generates) are
answered from the GPU-resident fp16 matrix by the exact score + top-k kernels; everything else (bm25, hybrid) is handed to the optional `delegate` — a real VespaClient — or rejected with VespaError (SURVEY §8b:
"delegate ... rather than answer").

Semantics implemented (from the schema generators the reference ships, executed inside Vespa today):
  score(doc) = max over searched tensor fields, max over chunks, of closeness(q, chunk)
               (unstructured_vespa_schema.py:225-230,292-294; structured_vespa_index.py:645-688)
  matchfeatures: closest(<embeddings field>) = arg-max chunk label, distance(field,<embeddings field>)
               (consumed by _extract_highlights, structured_vespa_index.py:942-1000)
  score modifiers: relevance = modify(score, query(marqo__mult_weights_tensor), query(marqo__add_weights_tensor))
               over the document's `marqo__score_modifiers` cells (unstructured_vespa_schema.py:225-230,266-271;
               vespa_index.py:106-150; unstructured_document.py:110-125), evaluated inside the scan kernel (f3)
"""
from __future__ import annotations

import math
import re
import threading
import time
from collections import OrderedDict
from typing import Any, Dict, List, Optional, Tuple

import numpy as np

from ._native import ERR_UNSUPPORTED, MAX_INDEX_DIM, NativeError
from .engine import RowStore
from .yql_filter import FilterSyntaxError, compile_filter
from .errors import VespaError, VespaStatusError

RANK_PROFILE_EMBEDDING_SIMILARITY = "embedding_similarity"   # */common.py
RANK_PROFILE_EMBEDDING_SIMILARITY_MODIFIERS_2_9 = "embedding_similarity_modifiers"   # */common.py (index version < 2.10)
SCORE_MODIFIERS_FIELD = "marqo__score_modifiers"             # */common.py SCORE_MODIFIERS
# structured indexes split the cells over two tensors whose products / sums are multiplied / added together
# (structured_vespa_index/common.py:3-5, structured_vespa_schema.py:256-262): one sparse tensor over their union
SCORE_MODIFIER_FIELDS = (SCORE_MODIFIERS_FIELD, "marqo__score_modifiers_float", "marqo__score_modifiers_double_long")
MULT_WEIGHTS_INPUTS = ("marqo__mult_weights_tensor", "marqo__mult_weights")   # core/constants.py:22-27
ADD_WEIGHTS_INPUTS = ("marqo__add_weights_tensor", "marqo__add_weights")
MAX_ATTRIBUTE_COLUMNS = 64
MAX_MODIFIER_TERMS = 16
QUERY_INPUT_EMBEDDINGS = ("marqo__query_embedding", "embedding_query")
EMBEDDINGS_PREFIX = "marqo__embeddings"
CHUNKS_PREFIX = "marqo__chunks"
MATCH_FEATURES = "matchfeatures"

ROW_ALIGN = 64   # the row store's width is a multiple of this; narrower fields are stored with zero columns appended


def _padded_width(dim: int) -> int:
    return -(-dim // ROW_ALIGN) * ROW_ALIGN


def _pad_columns(mat: np.ndarray, width: int) -> np.ndarray:
    """[m, d] -> [m, width] with zero columns appended.  Zero columns add exact zeros to every dot product, norm and
    fp64 re-score sum, so ids, rows and scores are those of the unpadded vectors."""
    if mat.shape[-1] == width:
        return mat
    out = np.zeros(mat.shape[:-1] + (width,), dtype=np.float32)
    out[..., :mat.shape[-1]] = mat
    return out


_NN_TERM = re.compile(r"\(\s*\{([^}]*)\}\s*nearestNeighbor\(\s*([A-Za-z0-9_]+)\s*,\s*([A-Za-z0-9_]+)\s*\)\s*\)")
_WHERE = re.compile(r"\bwhere\b(.*)$", re.IGNORECASE | re.DOTALL)


class _Obj:
    """Attribute bag with `.dict()` — stands in for the pydantic models where Marqo is not importable."""

    def __init__(self, **kw):
        self.__dict__.update(kw)

    def dict(self, **_):
        def conv(v):
            if isinstance(v, _Obj):
                return v.dict()
            if isinstance(v, list):
                return [conv(x) for x in v]
            return v
        return {k: conv(v) for k, v in self.__dict__.items()}


def _wrap_query_result(js: dict):
    try:  # real Marqo environment: return its own pydantic model
        from marqo.vespa.models import QueryResult  # type: ignore
        return QueryResult(**js)
    except Exception:
        root = js["root"]
        children = [_Obj(id=c["id"], relevance=c["relevance"], source=c.get("source"), fields=c["fields"])
                    for c in root.get("children", [])]
        cov = root["coverage"]
        coverage = _Obj(coverage=cov["coverage"], documents=cov["documents"], full=cov["full"], nodes=cov["nodes"],
                        results=cov["results"], results_full=cov["resultsFull"], degraded=None)
        r = _Obj(id=root["id"], relevance=root["relevance"], fields=_Obj(total_count=root["fields"]["totalCount"]),
                 coverage=coverage, children=children)
        out = _Obj(root=r, timing=None, trace=None)
        out.hits = children
        out.total_count = root["fields"]["totalCount"]
        return out


def _wrap(kind: str, js: dict):
    try:
        import marqo.vespa.models as vm  # type: ignore
        return getattr(vm, kind)(**js)
    except Exception:
        resp = []
        for r in js["responses"]:
            d = dict(r)
            if "fields" in d:
                d["document"] = _Obj(id=d.get("id"), fields=d.pop("fields"))
            else:
                d.setdefault("document", None)
            d["path_id"] = d.pop("pathId", None)
            d.setdefault("message", None)
            resp.append(_Obj(**d))
        return _Obj(responses=resp, errors=js["errors"])


class DeviceChunks:
    """Embeddings of one tensor field of one document that are ALREADY on the index's GPU (fp32 [n, dim], row-major):
    what the add_documents fast path puts in `fields['marqo__embeddings_<f>']` instead of {"0": [floats], ...}
    (semi_structured_document.py:139-141) so the vectors never visit the host.  `owner` keeps the device buffer alive
    (a torch tensor, or anything else) until feed_batch has copied the rows into the row store."""

    __slots__ = ("keys", "ptr", "dim", "owner")

    def __init__(self, keys: List[str], ptr: int, dim: int, owner=None):
        self.keys = [str(k) for k in keys]
        self.ptr = int(ptr)
        self.dim = int(dim)
        self.owner = owner


class _FilterEntry:
    __slots__ = ("keep", "bits", "tag", "packed")

    def __init__(self, keep):
        self.keep = keep
        self.bits = np.zeros(0, dtype=bool)    # per document number: may match
        self.tag = 0
        self.packed = None                     # uint32 bitset of `bits`, rebuilt lazily


class _Schema:
    def __init__(self):
        self.stores: Dict[str, RowStore] = {}          # embeddings field -> row store
        self.dims: Dict[str, int] = {}                 # embeddings field -> its vectors' dimension (<= store width)
        self.row_chunk: Dict[str, List[Tuple[int, str]]] = {}  # embeddings field -> row -> (doc number, chunk key)
        self.doc_num: Dict[str, int] = {}              # external id -> document number
        self.doc_ids: List[Optional[str]] = []         # document number -> external id (None = deleted)
        self.fields: List[Optional[dict]] = []         # document number -> stored non-vector fields
        self.doc_rows: List[Dict[str, List[int]]] = [] # document number -> field -> rows
        self.attr_col: Dict[str, int] = {}             # score-modifier attribute name -> device column
        self.attrs: List[Dict[str, float]] = []        # document number -> its marqo__score_modifiers cells
        self.dead: Dict[str, int] = {}                 # embeddings field -> tombstoned rows still in the matrix
        self.epoch = 0                                 # bumped when row numbers change (compaction)
        self.filters: "OrderedDict[str, _FilterEntry]" = OrderedDict()   # filter text -> document bitset (LRU)
        self.n_live = 0


class _Batch:
    __slots__ = ("queries", "ks", "done", "result", "error", "closed")

    def __init__(self):
        self.queries: List[np.ndarray] = []
        self.ks: List[int] = []
        self.done = threading.Event()
        self.result = None
        self.error = None
        self.closed = False


class _Coalescer:
    """Gathers concurrent single-query searches into one scan.  Marqo issues one `vespa_client.query()` per request
    (tensor_search.py:2189) from up to 8 concurrent search threads (api/configs.py:27-28); a corpus scan costs the same
    for 1 or 64 queries (the kernel is HBM-bound), so requests that arrive within a short window and agree on
    (row store, modifiers, filter) share a scan.  The first arrival leads: it waits `window_s` only when other requests
    are in flight, closes the batch, runs it, and hands every follower its slice."""

    def __init__(self, window_s: float = 0.0002, max_batch: int = 64):
        self.window_s = window_s
        self.max_batch = max_batch
        self._lock = threading.Lock()
        self._open: Dict[Any, _Batch] = {}
        self.active = 0            # requests currently inside GpuTensorIndex.query()
        self.batches = 0
        self.queries = 0

    def submit(self, key, q: np.ndarray, k: int, run):
        """run(Q [n, dim], kmax) -> (doc, row, score) arrays [n, kmax].  Returns this query's ([k], [k], [k])."""
        with self._lock:
            b = self._open.get(key)
            leader = b is None or b.closed or len(b.queries) >= self.max_batch
            if leader:
                b = _Batch()
                self._open[key] = b
            slot = len(b.queries)
            b.queries.append(q)
            b.ks.append(k)
            others = self.active > 1
        if not leader:
            b.done.wait()
            if b.error is not None:
                raise b.error
        else:
            if others and self.window_s > 0:
                deadline = time.perf_counter() + self.window_s
                while time.perf_counter() < deadline and len(b.queries) < self.max_batch:
                    time.sleep(self.window_s / 4)
            with self._lock:
                b.closed = True
                if self._open.get(key) is b:
                    del self._open[key]
                Q = np.stack(b.queries)
                kmax = max(b.ks)
                self.batches += 1
                self.queries += len(b.queries)
            try:
                b.result = run(Q, kmax)
            except BaseException as e:   # followers must not hang
                b.error = e
                b.done.set()
                raise
            b.done.set()
        doc, row, score = b.result
        return doc[slot, :k], row[slot, :k], score[slot, :k]


class GpuTensorIndex:
    COMPACT_MIN_DEAD = 4096        # compaction threshold: dead rows >= this AND >= COMPACT_DEAD_FRACTION of the matrix
    COMPACT_DEAD_FRACTION = 0.3
    MAX_CACHED_FILTERS = 32

    def __init__(self, metric: str = "prenormalized-angular", device: int = 0, delegate=None,
                 default_search_timeout_ms: int = 1000, coalesce_window_s: float = 0.0002):
        self.metric = metric
        self.device = device
        self.delegate = delegate
        self.default_search_timeout_ms = default_search_timeout_ms
        self._schemas: Dict[str, _Schema] = {}
        self._lock = threading.RLock()
        self._coalescer = _Coalescer(window_s=coalesce_window_s)
        self._next_tag = 1

    def close(self) -> None:
        with self._lock:
            for s in self._schemas.values():
                for st in s.stores.values():
                    st.close()
            self._schemas.clear()

    def coalescer_stats(self) -> Dict[str, int]:
        return {"batches": self._coalescer.batches, "queries": self._coalescer.queries}

    # ------------------------------------------------------------------------------------------------ feed
    @staticmethod
    def _doc_id_and_fields(doc) -> Tuple[str, dict]:
        if isinstance(doc, dict):
            return doc["id"], doc["fields"]
        return doc.id, doc.fields

    @staticmethod
    def _replay_attributes(s: _Schema, store: RowStore) -> None:
        """A row store created after documents were fed (a new tensor field) gets their attribute cells."""
        cols, ids, vals = [], [], []
        for num, attrs in enumerate(s.attrs):
            for name, v in attrs.items():
                cols.append(s.attr_col[name])
                ids.append(num)
                vals.append(v)
        if cols:
            store.set_attributes_multi(cols, ids, vals)

    def _fp16_limit(self) -> Optional[float]:
        # the angular metric L2-normalises rows at insert time: any finite vector fits; the others store values as given
        return None if self.metric == "angular" else 65504.0

    def _parse_document(self, s: _Schema, fields: dict, pending_cols: Dict[str, int]):
        """Everything that can reject a document, with NO side effect on the schema: -> (staged {field: (keys, mat |
        DeviceChunks)}, attrs).  Raises ValueError / KeyError / TypeError with the message for the 400 response."""
        staged = {}
        limit = self._fp16_limit()
        for f, cells in fields.items():
            if not f.startswith(EMBEDDINGS_PREFIX):
                continue
            if isinstance(cells, DeviceChunks):
                dim, keys, mat = cells.dim, cells.keys, cells
            else:
                if not isinstance(cells, dict):
                    raise ValueError(f"field {f}: expected a mapped tensor {{chunk: [floats]}}")
                keys = [str(k) for k in cells.keys()]
                mat = np.asarray([cells[k] for k in cells.keys()], dtype=np.float32)
                if mat.size and mat.ndim != 2:
                    raise ValueError(f"field {f}: ragged embeddings")
                if not len(keys):
                    continue
                if not np.isfinite(mat).all():
                    raise ValueError(f"field {f}: embedding values must be finite")
                if limit is not None and np.abs(mat).max() > limit:
                    raise ValueError(f"field {f}: embedding values beyond +-{limit:g} do not fit the fp16 row store")
                dim = mat.shape[1]
            store = s.stores.get(f)
            if store is not None and dim != s.dims[f]:
                raise ValueError(f"field {f}: embedding dimension {dim} != index dimension {s.dims[f]}")
            if store is None and not 0 < dim <= MAX_INDEX_DIM:
                raise ValueError(f"field {f}: embedding dimension {dim} is not in [1, {MAX_INDEX_DIM}]")
            if isinstance(mat, DeviceChunks) and dim != _padded_width(dim):
                raise ValueError(f"field {f}: device-resident embeddings of dimension {dim} are not a multiple of "
                                 f"{ROW_ALIGN}; send them as host vectors")
            staged[f] = (keys, mat)
        attrs: Dict[str, float] = {}
        for tensor_field in SCORE_MODIFIER_FIELDS:
            cells = fields.get(tensor_field) or {}
            if isinstance(cells, dict) and "cells" in cells and isinstance(cells["cells"], (dict, list)):
                cells = cells["cells"]          # Vespa's verbose tensor JSON form
            if isinstance(cells, list):
                cells = {c["address"]["p"]: c["value"] for c in cells}
            for name, v in cells.items():
                # structured indexes keep float-typed modifier fields in a tensor<float>: fp32 cells
                attrs[str(name)] = float(np.float32(v)) if tensor_field.endswith("_float") else float(v)
        new_cols = 0
        for name, v in attrs.items():
            if not math.isfinite(v):
                raise ValueError(f"score modifier field {name}: value {v} is not finite")
            if name not in s.attr_col and name not in pending_cols:
                new_cols += 1
        if len(s.attr_col) + len(pending_cols) + new_cols > MAX_ATTRIBUTE_COLUMNS:
            raise ValueError(f"more than {MAX_ATTRIBUTE_COLUMNS} distinct score-modifier fields")
        return staged, attrs

    def feed_batch(self, batch: List[Any], schema: str, concurrency: Optional[int] = None, timeout: int = 60):
        """vespa_client.py:267-296.  Embeddings arrive as fields['marqo__embeddings[_<field>]'] = {"0": [...], ...}
        (semi_structured_document.py:139-141; unstructured_add_document_handler.py:162-163) or, on the device fast
        path, as DeviceChunks.

        Two phases.  (1) every document is parsed and validated with no side effect; a rejected document gets its 400
        and leaves the index exactly as it was (Vespa leaves the old version of a failed put intact).  (2) the accepted
        documents are committed with ONE row append per tensor field, ONE tombstone scatter per field for the replaced
        versions and ONE attribute scatter per row store — no per-document device allocation or synchronisation.  A
        native failure in phase 2 (out of device memory, ...) undoes the host-side registration of the whole batch and
        is reported per document as a 507."""
        responses: List[Optional[dict]] = [None] * len(batch)
        errors = False
        with self._lock:
            s = self._schemas.setdefault(schema, _Schema())
            accepted = []            # (position, doc_id, fields, staged, attrs) in feed order
            pending_cols: Dict[str, int] = {}
            for pos, doc in enumerate(batch):
                doc_id, fields = None, None
                try:
                    doc_id, fields = self._doc_id_and_fields(doc)
                    staged, attrs = self._parse_document(s, fields, pending_cols)
                    for name in attrs:
                        if name not in s.attr_col and name not in pending_cols:
                            pending_cols[name] = len(s.attr_col) + len(pending_cols)
                    accepted.append((pos, doc_id, fields, staged, attrs))
                except (ValueError, KeyError, TypeError, AttributeError) as e:
                    errors = True
                    responses[pos] = {"status": 400, "pathId": f"/document/v1/{schema}/{schema}/docid/{doc_id}",
                                      "id": f"id:{schema}:{schema}::{doc_id}", "message": str(e)}
            # the LAST put of an id within the batch wins (Vespa applies puts in order); earlier ones succeed and vanish
            last_pos = {doc_id: pos for pos, doc_id, *_ in accepted}
            undo = self._commit(s, schema, [a for a in accepted if last_pos[a[1]] == a[0]], pending_cols)
            for pos, doc_id, *_ in accepted:
                status, msg = (200, None) if undo is None else (507, undo)
                errors = errors or undo is not None
                responses[pos] = {"status": status, "pathId": f"/document/v1/{schema}/{schema}/docid/{doc_id}",
                                  "id": f"id:{schema}:{schema}::{doc_id}", "message": msg}
        return _wrap("FeedBatchResponse", {"responses": responses, "errors": errors})

    def _commit(self, s: _Schema, schema: str, docs, pending_cols: Dict[str, int]) -> Optional[str]:
        """Phase 2 of feed_batch.  Returns None on success, else the failure text (the index is unchanged then, except
        for appended-but-tombstoned rows)."""
        if not docs:
            return None
        n_before = len(s.doc_ids)
        new_ids: List[str] = []
        nums: List[int] = []
        for _, doc_id, *_ in docs:
            num = s.doc_num.get(doc_id)
            if num is None:
                num = n_before + len(new_ids)
                new_ids.append(doc_id)
            nums.append(num)
        replaced = [n for n in nums if n < n_before]
        # ---- device work first; host maps are only touched once it has all succeeded
        appended: Dict[str, Tuple[int, int]] = {}        # field -> (first new row, count)
        created: List[str] = []
        try:
            per_field: Dict[str, list] = {}
            for (_, _, _, staged, _), num in zip(docs, nums):
                for f, (keys, mat) in staged.items():
                    per_field.setdefault(f, []).append((num, keys, mat))
            for f, items in per_field.items():
                store = s.stores.get(f)
                if store is None:
                    dim = items[0][2].dim if isinstance(items[0][2], DeviceChunks) else items[0][2].shape[1]
                    for _, _, m in items:
                        d = m.dim if isinstance(m, DeviceChunks) else m.shape[1]
                        if d != dim:
                            raise ValueError(f"field {f}: embedding dimension {d} != index dimension {dim}")
                    store = RowStore(_padded_width(dim), metric=self.metric, device=self.device)
                    s.stores[f] = store
                    s.dims[f] = dim
                    s.row_chunk[f] = []
                    s.dead[f] = 0
                    created.append(f)
                    self._replay_attributes(s, store)
                row0 = len(store)
                host_rows, host_ids = [], []
                dev_ptr, dev_ids = 0, []      # a run of DeviceChunks that are contiguous in device memory

                def flush_host():
                    nonlocal host_rows, host_ids
                    if host_rows:
                        store.add(np.concatenate(host_rows), np.concatenate(host_ids))
                        host_rows, host_ids = [], []

                def flush_dev():
                    nonlocal dev_ptr, dev_ids
                    if dev_ids:
                        store.add_device_docs(dev_ptr, np.asarray(dev_ids, dtype=np.int32))
                        dev_ptr, dev_ids = 0, []

                for num, keys, mat in items:       # rows are appended in feed order
                    if isinstance(mat, DeviceChunks):
                        flush_host()
                        if dev_ids and mat.ptr != dev_ptr + len(dev_ids) * store.dim * 4:
                            flush_dev()
                        if not dev_ids:
                            dev_ptr = mat.ptr
                        dev_ids.extend([num] * len(keys))      # the vectoriser hands out consecutive slices of one
                    else:                                      # tensor: a whole batch becomes ONE device append
                        flush_dev()
                        host_rows.append(_pad_columns(mat, store.dim))
                        host_ids.append(np.full(len(keys), num, dtype=np.int32))
                flush_host()
                flush_dev()
                appended[f] = (row0, len(store) - row0)
            # attribute cells: clear the replaced documents' old cells, then write the new ones (per row store)
            cols, ids, vals = [], [], []
            col_of = dict(s.attr_col)
            col_of.update(pending_cols)
            for (_, _, _, _, attrs), num in zip(docs, nums):
                for name, v in attrs.items():
                    cols.append(col_of[name])
                    ids.append(num)
                    vals.append(v)
            had_attrs = [n for n in replaced if s.attrs[n]]
            for store in s.stores.values():
                if had_attrs:
                    store.set_attributes(-1, had_attrs, None)
                if cols:
                    store.set_attributes_multi(cols, ids, vals)
            # tombstone the replaced versions' rows (all fields), one scatter per field
            for f, store in s.stores.items():
                old = [r for n in replaced for r in s.doc_rows[n].get(f, ())]
                if old:
                    store.delete_rows(old)
                    s.dead[f] = s.dead.get(f, 0) + len(old)
        except (NativeError, ValueError) as e:
            # undo: rows appended by this batch become tombstones; nothing else was changed on the host.  (Attribute
            # cells of replaced documents may have been rewritten: restore them from the host copy.)
            for f, (row0, cnt) in appended.items():
                try:
                    if cnt:
                        s.stores[f].delete_rows(np.arange(row0, row0 + cnt, dtype=np.int32))
                        s.row_chunk[f].extend((-1, "") for _ in range(cnt))
                        s.dead[f] = s.dead.get(f, 0) + cnt
                except NativeError:
                    pass
            for f in created:
                if f not in appended:
                    s.stores.pop(f).close()
                    s.dims.pop(f, None)
                    s.row_chunk.pop(f, None)
            try:
                rc, ri, rv = [], [], []
                for n in replaced:
                    for name, v in s.attrs[n].items():
                        rc.append(s.attr_col[name]); ri.append(n); rv.append(v)
                for store in s.stores.values():
                    if replaced:
                        store.set_attributes(-1, replaced, None)
                    if rc:
                        store.set_attributes_multi(rc, ri, rv)
            except NativeError:
                pass
            return str(getattr(e, "message", e))
        # ---- host registration (cannot fail)
        s.attr_col.update(pending_cols)
        for doc_id in new_ids:
            s.doc_num[doc_id] = len(s.doc_ids)
            s.doc_ids.append(doc_id)
            s.fields.append(None)
            s.doc_rows.append({})
            s.attrs.append({})
        s.n_live += len(new_ids)
        for n in replaced:
            s.doc_rows[n] = {}
        cursor = {f: row0 for f, (row0, _) in appended.items()}
        for (_, doc_id, fields, staged, attrs), num in zip(docs, nums):
            s.doc_ids[num] = doc_id
            for f, (keys, _) in staged.items():
                r0 = cursor[f]
                s.row_chunk[f].extend((num, k) for k in keys)
                s.doc_rows[num][f] = list(range(r0, r0 + len(keys)))
                cursor[f] = r0 + len(keys)
            s.fields[num] = {k: v for k, v in fields.items() if not k.startswith(EMBEDDINGS_PREFIX)}
            s.attrs[num] = attrs
        self._filters_update(s, nums)
        self._maybe_compact(s)
        return None

    def _maybe_compact(self, s: _Schema) -> None:
        """Tombstoned rows are squeezed out once they are a sizeable share of a matrix (update-heavy feeds would
        otherwise grow HBM use and scan time without bound)."""
        for f, store in s.stores.items():
            dead = s.dead.get(f, 0)
            rows = len(s.row_chunk[f])
            if dead < self.COMPACT_MIN_DEAD or dead < self.COMPACT_DEAD_FRACTION * rows:
                continue
            new_of_old = store.compact()
            rc = s.row_chunk[f]
            s.row_chunk[f] = [rc[i] for i in np.flatnonzero(new_of_old >= 0)]
            for num in range(len(s.doc_rows)):
                rows_f = s.doc_rows[num].get(f)
                if rows_f:
                    s.doc_rows[num][f] = [int(new_of_old[r]) for r in rows_f]
            s.dead[f] = 0
            s.epoch += 1

    # ------------------------------------------------------------------------------------------------ filters
    def _filter_entry(self, s: _Schema, text: str) -> _FilterEntry:
        """The document bitset of one filter string: compiled and evaluated over the schema ONCE, then kept current by
        feed_batch / delete_batch (only the touched documents are re-evaluated)."""
        e = s.filters.get(text)
        if e is None:
            e = _FilterEntry(compile_filter(text))
            n = len(s.doc_ids)
            e.bits = np.fromiter((d is not None and bool(e.keep(s.fields[i] or {})) for i, d in enumerate(s.doc_ids)),
                                 dtype=bool, count=n)
            e.tag = self._take_tag()
            s.filters[text] = e
            while len(s.filters) > self.MAX_CACHED_FILTERS:
                s.filters.popitem(last=False)
        else:
            s.filters.move_to_end(text)
        return e

    def _take_tag(self) -> int:
        self._next_tag += 1
        return self._next_tag

    def _filters_update(self, s: _Schema, nums: List[int]) -> None:
        if not s.filters or not nums:
            return
        n = len(s.doc_ids)
        for e in s.filters.values():
            if len(e.bits) < n:
                e.bits = np.concatenate([e.bits, np.zeros(n - len(e.bits), dtype=bool)])
            for num in nums:
                e.bits[num] = s.doc_ids[num] is not None and bool(e.keep(s.fields[num] or {}))
            e.tag = self._take_tag()
            e.packed = None

    @staticmethod
    def _packed(e: _FilterEntry) -> np.ndarray:
        if e.packed is None:
            b = np.packbits(e.bits, bitorder="little")
            pad = (-len(b)) % 4
            if pad:
                b = np.concatenate([b, np.zeros(pad, np.uint8)])
            e.packed = b.view(np.uint32) if len(b) else np.zeros(1, np.uint32)
        return e.packed

    # ------------------------------------------------------------------------------------------------ query
    @staticmethod
    def _split_where(yql: str) -> Tuple[bool, Optional[str]]:
        """-> (the where clause is nearestNeighbor terms [AND <filter>], filter text or None).
        unstructured_vespa_index.py:59-66: `where {tensor_term}{' AND ' + filter}`; structured_vespa_index.py:645-688 ORs
        one nearestNeighbor term per searched field inside parentheses."""
        m = _WHERE.search(yql or "")
        if not m:
            return False, None
        rest = _NN_TERM.sub("", m.group(1))
        head, sep, tail = rest.partition(" AND ")
        if re.sub(r"\bOR\b|[()\s;]", "", head):
            return False, None
        if not sep:
            return True, None
        text = tail.strip().rstrip(";").strip()
        return (True, text) if text else (False, None)

    def _is_tensor_query(self, yql: str, ranking: Optional[str], query_features: Optional[dict]) -> bool:
        if ranking not in (RANK_PROFILE_EMBEDDING_SIMILARITY, RANK_PROFILE_EMBEDDING_SIMILARITY_MODIFIERS_2_9):
            return False
        ok, filter_text = self._split_where(yql)
        if not ok:
            return False
        if filter_text is not None:
            try:
                compile_filter(filter_text)
            except FilterSyntaxError:     # text neither of the reference's filter generators emits: not ours to answer
                return False
        qf = query_features or {}
        if not any(k in qf for k in QUERY_INPUT_EMBEDDINGS):
            return False
        for k, v in qf.items():   # lexical / global modifier tensors belong to other rank profiles
            if (k.startswith("marqo__mult_weights") or k.startswith("marqo__add_weights")) and \
                    k not in MULT_WEIGHTS_INPUTS + ADD_WEIGHTS_INPUTS and v:
                return False
        n_mult = sum(len(qf.get(k) or {}) for k in MULT_WEIGHTS_INPUTS)
        n_add = sum(len(qf.get(k) or {}) for k in ADD_WEIGHTS_INPUTS)
        return n_mult <= MAX_MODIFIER_TERMS and n_add <= MAX_MODIFIER_TERMS

    def query(self, yql: str, hits: int = 10, ranking: str = None, model_restrict: str = None,
              query_features: Dict[str, Any] = None, timeout: float = None, **kwargs):
        """vespa_client.py:198-242."""
        if not self._is_tensor_query(yql, ranking, query_features):
            if self.delegate is not None:
                return self.delegate.query(yql, hits=hits, ranking=ranking, model_restrict=model_restrict,
                                           query_features=query_features, timeout=timeout, **kwargs)
            raise VespaError("GpuTensorIndex only answers exact tensor queries (ranking=embedding_similarity, "
                             "nearestNeighbor terms only); no delegate VespaClient is configured")
        schema = model_restrict
        if schema is None:
            m = re.search(r"\bfrom\s+([A-Za-z0-9_]+)", yql)
            schema = m.group(1) if m else None
        offset = int(kwargs.get("offset", 0) or 0)
        terms = _NN_TERM.findall(yql)
        fields = [t[1] for t in terms]
        qname = next(k for k in QUERY_INPUT_EMBEDDINGS if k in query_features)
        q = np.asarray(query_features[qname], dtype=np.float32)
        mult: Dict[str, float] = {}
        add: Dict[str, float] = {}
        for k in MULT_WEIGHTS_INPUTS:
            mult.update(self._weights(query_features.get(k)))
        for k in ADD_WEIGHTS_INPUTS:
            add.update(self._weights(query_features.get(k)))
        filter_text = self._split_where(yql)[1]
        co = self._coalescer
        with co._lock:
            co.active += 1
        try:
            s = self._schemas.get(schema)
            children, n_docs = [], 0
            if s is not None:
                try:
                    children, n_docs = self._search(s, schema, fields, q, hits, offset, mult, add, filter_text)
                except NativeError as e:
                    if e.code != ERR_UNSUPPORTED:
                        raise
                    if self.delegate is not None:
                        return self.delegate.query(yql, hits=hits, ranking=ranking, model_restrict=model_restrict,
                                                   query_features=query_features, timeout=timeout, **kwargs)
                    raise VespaError(f"GpuTensorIndex cannot answer this query: {e.message}") from e
        finally:
            with co._lock:
                co.active -= 1
        js = {"root": {"id": "toplevel", "relevance": 1.0, "fields": {"totalCount": len(children) + offset},
                       "coverage": {"coverage": 100, "documents": n_docs, "full": True, "nodes": 1, "results": 1,
                                    "resultsFull": 1},
                       "children": children}}
        return _wrap_query_result(js)

    @staticmethod
    def _weights(tensor) -> Dict[str, float]:
        """A query tensor<double>(p{}) as Marqo sends it ({field: weight}) or in Vespa's {"cells": ...} forms."""
        if not tensor:
            return {}
        if isinstance(tensor, dict) and "cells" in tensor:
            tensor = tensor["cells"]
        if isinstance(tensor, list):
            return {c["address"]["p"]: float(c["value"]) for c in tensor}
        return {str(k): float(v) for k, v in tensor.items()}

    @staticmethod
    def _modifier_of(attrs: Dict[str, float], mult: Dict[str, float], add: Dict[str, float]) -> Tuple[float, float]:
        """(multiplier, addend) of one document — the host copy of the device table, used to recover the raw
        closeness for the distance() match-feature."""
        m, cnt = 1.0, 0
        for name, w in mult.items():
            if name in attrs:
                m *= w * attrs[name]
                cnt += 1
        if cnt == 0:
            m = 1.0
        a = 0.0
        for name, w in add.items():
            if name in attrs:
                a += w * attrs[name]
        return m, a

    MAX_FETCH = 11000   # b200_index_search's own k limit (Marqo's limit + offset cap, api/configs.py:24-25)

    def _search(self, s: _Schema, schema: str, fields: List[str], q: np.ndarray, hits: int, offset: int,
                mult: Optional[Dict[str, float]] = None, add: Optional[Dict[str, float]] = None,
                filter_text: Optional[str] = None) -> Tuple[List[dict], int]:
        k = hits + offset
        if k <= 0:
            return [], s.n_live
        if k > self.MAX_FETCH:
            raise VespaStatusError(400, f"hits + offset = {k} exceeds {self.MAX_FETCH}")
        for attempt in range(4):
            found: Dict[str, tuple] = {}
            epoch = None
            for f in fields:
                with self._lock:
                    store = s.stores.get(f)
                    if store is None or len(store) == 0:
                        continue
                    if q.shape[-1] != s.dims[f]:
                        raise VespaStatusError(400, f"Expected a tensor of dimension {s.dims[f]} for query input but "
                                                    f"got {q.shape[-1]}")
                    qf = _pad_columns(q, store.dim)
                    if epoch is None:
                        epoch = s.epoch
                    # a weight on an attribute no document has multiplies / adds nothing anywhere: drop the term
                    mult_cols = tuple((s.attr_col[n], w) for n, w in (mult or {}).items() if n in s.attr_col)
                    add_cols = tuple((s.attr_col[n], w) for n, w in (add or {}).items() if n in s.attr_col)

                def run(Q, kmax, store=store, mult_cols=mult_cols, add_cols=add_cols):
                    # the leader of a batch runs the scan for everybody, under the index lock (no concurrent mutation)
                    with self._lock:
                        kw = {}
                        if filter_text is not None:
                            e = self._filter_entry(s, filter_text)
                            kw = dict(filter_bits=self._packed(e), filter_docs=len(e.bits), filter_tag=e.tag)
                        return store.search(Q, kmax, mult=mult_cols, add=add_cols, **kw)

                key = (id(store), mult_cols, add_cols, filter_text)
                found[f] = self._coalescer.submit(key, qf, k, run)
            with self._lock:
                if epoch is not None and epoch != s.epoch:
                    continue      # a compaction renumbered rows between the scan and now: search again
                return self._children(s, schema, found, hits, offset, mult, add), s.n_live
        raise VespaError("the index kept changing under the query")

    def _children(self, s: _Schema, schema: str, found: Dict[str, tuple], hits: int, offset: int, mult, add) -> List[dict]:
        modified = bool(mult) or bool(add)
        best: Dict[int, Tuple[float, str, int]] = {}   # doc number -> (score, field, row)
        for f, (doc, row, score) in found.items():
            for d, r, sc in zip(doc.tolist(), row.tolist(), score.tolist()):
                if d < 0:
                    continue
                cur = best.get(d)
                if cur is None or sc > cur[0]:
                    best[d] = (sc, f, r)
        ranked = sorted(best.items(), key=lambda kv: (-kv[1][0], kv[0]))[offset:offset + hits]
        children = []
        for num, (sc, f, r) in ranked:
            chunk_key = s.row_chunk[f][r][1]
            out_fields = dict(s.fields[num] or {})
            raw = sc
            if modified:   # relevance is the modified score; distance() stays the raw one
                m, a = self._modifier_of(s.attrs[num], mult or {}, add or {})
                raw = (sc - a) / m if m != 0 else float("nan")
            out_fields[MATCH_FEATURES] = {
                f"closest({f})": {"type": "tensor<float>(p{})", "cells": {chunk_key: 1.0}},
                f"distance(field,{f})": self._distance_from_closeness(raw),
            }
            children.append({"id": f"id:{schema}:{schema}::{s.doc_ids[num]}", "relevance": sc, "source": "content_default",
                             "fields": out_fields})
        return children

    def _distance_from_closeness(self, closeness: float) -> float:
        if self.metric == "dotproduct":
            return -closeness
        return 1.0 / closeness - 1.0 if closeness > 0 else math.inf

    # ------------------------------------------------------------------------------------------------ get / delete
    def get_batch(self, ids: List[str], schema: str, concurrency: Optional[int] = None, timeout: int = 60,
                  fields: Optional[List[str]] = None):
        """vespa_client.py:405-440: 404 entries are returned, not raised.  Embeddings are read back from the fp16
        row store (use_existing_tensors, add_documents_handler.py:160-165)."""
        responses = []
        with self._lock:
            s = self._schemas.get(schema)
            for doc_id in ids:
                path_id = f"/document/v1/{schema}/{schema}/docid/{doc_id}"
                num = s.doc_num.get(doc_id) if s else None
                if num is None or s.doc_ids[num] is None:
                    responses.append({"status": 404, "pathId": path_id, "id": f"id:{schema}:{schema}::{doc_id}",
                                      "message": "Document not found"})
                    continue
                out = dict(s.fields[num] or {})
                for f, rows in s.doc_rows[num].items():
                    if rows:
                        vecs = s.stores[f].get_rows(rows)[:, :s.dims[f]]
                        out[f] = {s.row_chunk[f][r][1]: vecs[i].tolist() for i, r in enumerate(rows)}
                if fields is not None:
                    out = {k: v for k, v in out.items() if k in fields}
                responses.append({"status": 200, "pathId": path_id, "id": f"id:{schema}:{schema}::{doc_id}",
                                  "fields": out})
        return _wrap("GetBatchResponse", {"responses": responses, "errors": False})

    def delete_batch(self, ids: List[str], schema: str, concurrency: Optional[int] = None, timeout: int = 60):
        """vespa_client.py:468-500 (deleting a missing id is a 200 in Vespa's document API)."""
        responses = []
        with self._lock:
            s = self._schemas.get(schema)
            gone: List[int] = []
            for doc_id in ids:
                num = s.doc_num.get(doc_id) if s else None
                if num is not None and s.doc_ids[num] is not None and num not in gone:
                    gone.append(num)
                responses.append({"status": 200, "pathId": f"/document/v1/{schema}/{schema}/docid/{doc_id}",
                                  "id": f"id:{schema}:{schema}::{doc_id}", "message": None})
            if gone:    # one tombstone scatter per tensor field, one attribute clear per row store
                for f, store in s.stores.items():
                    rows = [r for n in gone for r in s.doc_rows[n].get(f, ())]
                    if rows:
                        store.delete_rows(rows)
                        s.dead[f] = s.dead.get(f, 0) + len(rows)
                with_attrs = [n for n in gone if s.attrs[n]]
                if with_attrs:
                    for store in s.stores.values():
                        store.set_attributes(-1, with_attrs, None)
                for num in gone:
                    del s.doc_num[s.doc_ids[num]]
                    s.doc_ids[num] = None
                    s.fields[num] = None
                    s.doc_rows[num] = {}
                    s.attrs[num] = {}
                s.n_live -= len(gone)
                self._filters_update(s, gone)
                self._maybe_compact(s)
        return _wrap("DeleteBatchResponse", {"responses": responses, "errors": False})

    # ------------------------------------------------------------------------------------------------ persistence
    def save(self, directory: str) -> None:
        """Corpus persistence (SURVEY §8 f4): one binary row-store snapshot per (schema, tensor field) —
        b200_index_save: fp16 rows + row -> document map + score-modifier columns — plus a JSON manifest with what
        Vespa would keep per document (ids, stored fields, chunk keys).  Restart = GpuTensorIndex.load(directory)."""
        import json
        import os
        os.makedirs(directory, exist_ok=True)
        manifest = {"format": 1, "metric": self.metric, "schemas": {}}
        with self._lock:
            for name, s in self._schemas.items():
                stores = {}
                for i, (f, st) in enumerate(sorted(s.stores.items())):
                    fname = f"{len(manifest['schemas'])}_{i}.b200idx"
                    st.save(os.path.join(directory, fname))
                    stores[f] = {"file": fname, "row_chunk": s.row_chunk[f]}
                    if s.dims[f] != st.dim:   # stored with zero columns appended
                        stores[f]["dim"] = s.dims[f]
                manifest["schemas"][name] = {"stores": stores, "doc_ids": s.doc_ids, "fields": s.fields,
                                             "doc_rows": s.doc_rows, "attr_col": s.attr_col, "attrs": s.attrs}
            tmp = os.path.join(directory, "manifest.json.tmp")
            with open(tmp, "w", encoding="utf-8") as fh:
                json.dump(manifest, fh)
            os.replace(tmp, os.path.join(directory, "manifest.json"))

    @classmethod
    def load(cls, directory: str, device: int = 0, delegate=None) -> "GpuTensorIndex":
        import json
        import os
        with open(os.path.join(directory, "manifest.json"), encoding="utf-8") as fh:
            manifest = json.load(fh)
        if manifest.get("format") != 1:
            raise VespaError(f"{directory}: unknown GpuTensorIndex snapshot format {manifest.get('format')!r}")
        ix = cls(metric=manifest["metric"], device=device, delegate=delegate)
        for name, js in manifest["schemas"].items():
            s = _Schema()
            s.doc_ids = list(js["doc_ids"])
            s.doc_num = {d: i for i, d in enumerate(s.doc_ids) if d is not None}
            s.fields = list(js["fields"])
            s.doc_rows = [{f: list(r) for f, r in d.items()} for d in js["doc_rows"]]
            s.attr_col = {k: int(v) for k, v in js["attr_col"].items()}
            s.attrs = [dict(a) for a in js["attrs"]]
            for f, st in js["stores"].items():
                s.stores[f] = RowStore.load(os.path.join(directory, st["file"]), device=device)
                s.dims[f] = int(st.get("dim", s.stores[f].dim))
                s.row_chunk[f] = [(int(n), str(k)) for n, k in st["row_chunk"]]
                live = sum(len(d.get(f, ())) for d in s.doc_rows)
                s.dead[f] = len(s.row_chunk[f]) - live
            s.n_live = sum(1 for d in s.doc_ids if d is not None)
            ix._schemas[name] = s
        return ix

    def get_document_count(self, schema: str) -> int:
        with self._lock:
            s = self._schemas.get(schema)
            return 0 if s is None else s.n_live


def gather_documents_from_response(response, tensor_fields_by_embeddings_field: Optional[Dict[str, str]] = None,
                                   highlights: bool = True) -> Dict[str, Any]:
    """Hit -> Marqo document (`_id`, stored fields, `_score`, `_highlights`): the arithmetic-free part of
    src/marqo/tensor_search/tensor_search.py:1771-1791 and structured_vespa_index.py:942-1000 for this adapter's
    QueryResult (a9).  `tensor_fields_by_embeddings_field` maps 'marqo__embeddings_<f>' -> marqo field name; the
    default strips the prefix."""
    hits = []
    for child in response.hits:
        fields = child.dict()["fields"] if hasattr(child, "dict") else child["fields"]
        doc = {k: v for k, v in fields.items() if not k.startswith("marqo__") and k != MATCH_FEATURES}
        doc["_id"] = child.id.split("::")[-1]
        doc["_score"] = child.relevance
        if highlights:
            mf = fields.get(MATCH_FEATURES, {})
            best = None
            for key, val in mf.items():
                if key.startswith("closest(") and val.get("cells"):
                    emb = key[len("closest("):-1]
                    dist = mf.get(f"distance(field,{emb})")
                    if best is None or dist < best[0]:
                        best = (dist, emb, next(iter(val["cells"])))
            doc["_highlights"] = []
            if best is not None:
                _, emb, chunk_key = best
                suffix = emb[len(EMBEDDINGS_PREFIX):]
                chunks = fields.get(CHUNKS_PREFIX + suffix)
                name = (tensor_fields_by_embeddings_field or {}).get(emb, suffix.lstrip("_") or emb)
                if chunks is not None:
                    doc["_highlights"] = [{name: chunks[int(chunk_key)]}]
        hits.append(doc)
    return {"hits": hits}
