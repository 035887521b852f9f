"""The score path's settle rules and its add entry points, pinned end to end.

- A query that matches a run of identical rows cannot be resolved by the merge guard, so it goes through the collect
  pass.  4000 collected rows fit the device finalize (FIN_CAP = 4096 rows per query); 5000 do not and are finalized on
  the host.  Both sides must give the oracle's exact top-k under every metric.
- b200_index_add, _add_device and _add_device_docs must leave the same index for the same rows, and must keep nothing of
  a batch they reject.
"""
import numpy as np
import pytest

import _checks as K

pytestmark = pytest.mark.gpu

METRICS = ("prenormalized-angular", "angular", "dotproduct", "euclidean")
DIM = 128
NAN_MSG = ("embeddings contain a value that is not finite or does not fit the fp16 row store (|x| <= 65504 after "
           "normalisation)")


def _tie_corpus(run, seed=0):
    """`run` identical rows (the first query's best match) among 8000 random unit rows; queries: that row and two
    random ones."""
    rng = np.random.default_rng(seed)
    corpus = K.unit_rows(rng, 8000 + run, DIM)
    start = 3000
    corpus[start:start + run] = corpus[start]
    q = np.concatenate([corpus[start:start + 1], K.unit_rows(rng, 2, DIM)])
    return corpus, q


@pytest.mark.parametrize("run", [4000, 5000], ids=["device-finalize", "host-finalize"])
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("chunks", [1, 2])
def test_tied_run_both_sides_of_finalize_capacity(gpu_required, score_oracle, run, metric, chunks):
    from marqo_b200.engine import RowStore
    corpus, q = _tie_corpus(run)
    doc_of_row = (np.arange(corpus.shape[0]) // chunks).astype(np.int32) if chunks > 1 else None
    store = RowStore(DIM, metric)
    try:
        store.add(corpus, doc_of_row)
        for k in (10, 1000, 4999):
            before = store.search_stats()["collect_passes"]
            K.assert_topk_equal(store.search(q, k), score_oracle.search(q, corpus, k, metric, doc_of_row))
            assert store.search_stats()["collect_passes"] >= before + 1
    finally:
        store.close()


@pytest.mark.parametrize("run", [4000, 5000], ids=["device-finalize", "host-finalize"])
def test_tied_run_with_score_modifiers(gpu_required, score_oracle, run):
    from marqo_b200.engine import RowStore
    metric = "prenormalized-angular"
    corpus, q = _tie_corpus(run, seed=1)
    doc_of_row = (np.arange(corpus.shape[0]) // 2).astype(np.int32)
    n_docs = int(doc_of_row.max()) + 1
    rng = np.random.default_rng(2)
    attrs = np.stack([rng.uniform(0.5, 2.0, n_docs), rng.uniform(-0.1, 0.1, n_docs)])
    attrs[1, 100:600] = np.nan                   # documents without the additive attribute
    attrs[:, 1500:1500 + run // 2] = [[1.25], [0.05]]   # the run's documents tie exactly under the modifiers too
    mult, add = [(0, 1.0)], [(1, 0.5)]
    store = RowStore(DIM, metric)
    try:
        store.add(corpus, doc_of_row)
        for c in range(2):
            ids = np.nonzero(~np.isnan(attrs[c]))[0].astype(np.int32)
            store.set_attributes(c, ids, attrs[c, ids])
        mod = score_oracle.modifiers(attrs, mult, add)
        for k in (10, 1000):
            before = store.search_stats()["collect_passes"]
            got = store.search_modified(q, k, mult, add)
            K.assert_topk_equal(got, score_oracle.search_modified(q, corpus, k, mod, metric, doc_of_row))
            assert store.search_stats()["collect_passes"] >= before + 1
    finally:
        store.close()


# ---------------------------------------------------------------------------------------------------- add paths
M = 70000   # more than one 64 Ki-row staging chunk of the host add


def _add_corpus():
    rng = np.random.default_rng(5)
    vecs = K.unit_rows(rng, M, DIM)
    ids = rng.permutation(M // 2).astype(np.int32)[np.arange(M) // 2]   # two chunks per document, shuffled numbers
    return vecs, ids


def _fill(store, path, vecs, ids):
    import torch
    d_v = torch.from_numpy(vecs).cuda()
    d_i = torch.from_numpy(ids).cuda()
    if path == "add_ids":
        store.add(vecs, ids)
    elif path == "add":
        store.add(vecs)
    elif path == "add_device_ids":
        store.add_device(d_v.data_ptr(), vecs.shape[0], d_i.data_ptr())
    elif path == "add_device":
        store.add_device(d_v.data_ptr(), vecs.shape[0])
    else:
        store.add_device_docs(d_v.data_ptr(), ids)
    torch.cuda.synchronize()


def _snapshot(store, q, tmp_path, name):
    rows = np.random.default_rng(6).choice(M, size=2000, replace=False)
    res = [store.get_rows(rows).tobytes()]
    for k in (10, 300):
        res += [a.tobytes() for a in store.search(q, k)]
    f = tmp_path / f"{name}.idx"
    store.save(str(f))
    res.append(f.read_bytes())
    return res


def test_every_add_path_leaves_the_same_index(gpu_required, tmp_path):
    from marqo_b200.engine import RowStore
    vecs, ids = _add_corpus()
    q = K.unit_rows(np.random.default_rng(7), 5, DIM)
    snaps = {}
    for path in ("add_ids", "add_device_ids", "add_device_docs", "add", "add_device"):
        store = RowStore(DIM)
        try:
            _fill(store, path, vecs, ids)
            assert len(store) == M
            snaps[path] = _snapshot(store, q, tmp_path, path)
        finally:
            store.close()
    assert snaps["add_device_ids"] == snaps["add_ids"]
    assert snaps["add_device_docs"] == snaps["add_ids"]
    assert snaps["add_device"] == snaps["add"]
    assert snaps["add"] != snaps["add_ids"]


BAD_BATCHES = {
    "nan": (NAN_MSG, lambda v, i: (v.__setitem__((3, 5), np.nan), i)),
    "above-fp16": (NAN_MSG, lambda v, i: (v.__setitem__((7, 0), 65600.0), i)),
    "negative-id": ("doc_ids[4] is negative", lambda v, i: (None, i.__setitem__(4, -2))),
}
HOST_ID_PATHS = ("add_ids", "add_device_docs")


@pytest.mark.parametrize("path", ["add_ids", "add", "add_device_ids", "add_device", "add_device_docs"])
def test_rejected_batch_leaves_nothing_behind(gpu_required, path):
    from marqo_b200 import _native as N
    from marqo_b200.engine import RowStore
    rng = np.random.default_rng(8)
    base, base_ids = K.unit_rows(rng, 500, DIM), np.arange(500, dtype=np.int32)
    q = K.unit_rows(rng, 3, DIM)
    store = RowStore(DIM, "dotproduct")
    try:
        _fill(store, path, base, base_ids)
        want = store.search(q, 20)
        for kind, (msg, spoil) in BAD_BATCHES.items():
            if kind == "negative-id" and path not in HOST_ID_PATHS:
                continue
            vecs, ids = K.unit_rows(rng, 40, DIM), np.arange(500, 540, dtype=np.int32)
            spoil(vecs, ids)
            with pytest.raises(N.NativeError) as e:
                _fill(store, path, vecs, ids)
            assert (e.value.code, e.value.message) == (N.ERR_INVALID_ARG, msg), kind
            assert len(store) == 500
            got = store.search(q, 20)
            for a, b in zip(got, want):
                np.testing.assert_array_equal(a, b)
        _fill(store, path, K.unit_rows(rng, 40, DIM), np.arange(500, 540, dtype=np.int32))
        assert len(store) == 540
    finally:
        store.close()
