"""GPU parity tests for score modifiers (SURVEY §8 f3): `modify(closeness, mult_weights, add_weights)` evaluated inside
the scan kernel, through the C ABI (b200_index_set_attributes / b200_index_search_modified), against
oracle/score_oracle.c's restatement of unstructured_vespa_schema.py:266-271.

Bar: doc ids and arg-max rows bit-exact; modified scores equal to 1e-12 (fp64, same operation order).
"""
import numpy as np
import pytest

import _checks as K

pytestmark = pytest.mark.gpu


def _attrs(rng, n_cols, n_docs, coverage=0.7, lo=0.0, hi=3.0):
    a = rng.uniform(lo, hi, size=(n_cols, n_docs))
    a[rng.random((n_cols, n_docs)) > coverage] = np.nan
    return a


def _feed_attrs(store, attrs):
    for c in range(attrs.shape[0]):
        ids = np.nonzero(~np.isnan(attrs[c]))[0].astype(np.int32)
        store.set_attributes(c, ids, attrs[c, ids])


def _search_modified(store, so, q, corpus, k, attrs, mult, add, metric="prenormalized-angular", doc_of_row=None):
    """(the store's, the oracle's) top-k of the same modified search."""
    got = store.search_modified(q, k, mult, add)
    return got, so.search_modified(q, corpus, k, so.modifiers(attrs, mult, add), metric, doc_of_row)


@pytest.mark.parametrize("n,d,nq,k", [(300, 64, 3, 5), (20000, 128, 5, 10), (50000, 768, 64, 10), (4097, 384, 70, 10)])
def test_modified_topk_matches_oracle(gpu_required, score_oracle, n, d, nq, k):
    from marqo_b200.engine import RowStore
    rng = np.random.default_rng(n + d)
    corpus = K.unit_rows(rng, n, d)
    q = K.unit_rows(rng, nq, d)
    attrs = _attrs(rng, 3, n)
    store = RowStore(d)
    store.add(corpus)
    _feed_attrs(store, attrs)
    doc, _, _ = K.assert_topk_equal(*_search_modified(store, score_oracle, q, corpus, k, attrs, [(0, 1.5), (1, 0.25)],
                                                      [(2, 0.3)]))
    # the modifiers really re-rank: the unmodified top-k differs
    plain, _, _ = store.search(q, k)
    assert not np.array_equal(doc, plain)
    # add-only and mult-only
    K.assert_topk_equal(*_search_modified(store, score_oracle, q, corpus, k, attrs, [], [(2, 0.3), (0, -0.05)]))
    K.assert_topk_equal(*_search_modified(store, score_oracle, q, corpus, k, attrs, [(1, 2.0)], []))
    # no terms at all == plain search (multiplier 1, addend 0)
    K.assert_topk_equal(store.search_modified(q, k, [], []), store.search(q, k), atol=1e-15)


def test_missing_cells_and_unset_columns(gpu_required, score_oracle):
    """count(mult * attr) == 0 -> multiplier 1; a column nobody ever set is missing everywhere."""
    from marqo_b200.engine import RowStore
    rng = np.random.default_rng(3)
    n, d = 5000, 128
    corpus = K.unit_rows(rng, n, d)
    q = K.unit_rows(rng, 4, d)
    attrs = np.full((6, n), np.nan)
    attrs[0, ::2] = rng.uniform(0.5, 2.0, size=n // 2)   # only even documents carry attribute 0
    store = RowStore(d)
    store.add(corpus)
    _feed_attrs(store, attrs)
    K.assert_topk_equal(*_search_modified(store, score_oracle, q, corpus, 10, attrs, [(0, 3.0), (5, 7.0)], [(4, 1.0)]))
    # zero attribute value -> product 0 -> score == addend only
    attrs[1, :] = 0.0
    store.set_attributes(1, np.arange(n, dtype=np.int32), attrs[1])
    doc, _, score = K.assert_topk_equal(*_search_modified(store, score_oracle, q, corpus, 10, attrs, [(1, 5.0)],
                                                          [(0, 1.0)]))
    assert np.all(score[doc >= 0] >= 0.0)
    # removing cells
    store.set_attributes(0, np.arange(0, n, 4, dtype=np.int32), None)
    attrs[0, 0:n:4] = np.nan
    K.assert_topk_equal(*_search_modified(store, score_oracle, q, corpus, 10, attrs, [(0, 3.0)], [(0, 0.5)]))
    store.set_attributes(-1, np.arange(100, dtype=np.int32), None)
    attrs[:, :100] = np.nan
    K.assert_topk_equal(*_search_modified(store, score_oracle, q, corpus, 10, attrs, [(0, 3.0)], [(1, 0.5)]))


@pytest.mark.parametrize("metric", ["angular", "dotproduct", "euclidean"])
def test_modified_other_metrics_and_chunks(gpu_required, score_oracle, metric):
    from marqo_b200.engine import RowStore
    rng = np.random.default_rng(17)
    n, d = 6000, 256
    corpus = rng.standard_normal((n, d)).astype(np.float32)
    q = rng.standard_normal((7, d)).astype(np.float32)
    doc_of_row = (np.arange(n) // 3).astype(np.int32)      # 3 chunks per document
    attrs = _attrs(rng, 2, n // 3, coverage=0.8, lo=0.1, hi=2.0)
    store = RowStore(d, metric=metric)
    store.add(corpus, doc_of_row)
    _feed_attrs(store, attrs)
    atol = 1e-9 if metric == "angular" else 1e-12       # acos differs in the last ulps between libm and CUDA
    for k in (10, 37):   # 37: multi-round
        K.assert_topk_equal(*_search_modified(store, score_oracle, q, corpus, k, attrs, [(0, 1.25)], [(1, 0.01)],
                                              metric, doc_of_row), atol=atol)


def test_negative_multiplier(gpu_required, score_oracle):
    from marqo_b200 import _native as N
    from marqo_b200.engine import RowStore
    rng = np.random.default_rng(23)
    n, d = 4000, 128
    corpus = K.unit_rows(rng, n, d)
    q = K.unit_rows(rng, 3, d)
    attrs = _attrs(rng, 1, n, coverage=0.5, lo=0.5, hi=1.5)
    store = RowStore(d)
    store.add(corpus)                       # one chunk per document: the best chunk is THE chunk, any sign works
    _feed_attrs(store, attrs)
    K.assert_topk_equal(*_search_modified(store, score_oracle, q, corpus, 10, attrs, [(0, -1.0)], []))
    chunks = RowStore(d)
    chunks.add(corpus, (np.arange(n) // 2).astype(np.int32))
    _feed_attrs(chunks, attrs[:, : n // 2])
    with pytest.raises(N.NativeError) as e:
        chunks.search_modified(q, 10, [(0, -1.0)], [])
    assert e.value.code == N.ERR_UNSUPPORTED
    chunks.search_modified(q, 10, [(0, 1.0)], [(0, -1.0)])     # negative ADDEND is fine


def test_modifier_argument_errors(gpu_required):
    from marqo_b200 import _native as N
    from marqo_b200.engine import RowStore
    store = RowStore(64)
    store.add(np.eye(64, dtype=np.float32))
    q = np.eye(64, dtype=np.float32)[:1]
    with pytest.raises(N.NativeError):
        store.set_attributes(64, [0], [1.0])
    with pytest.raises(N.NativeError):
        store.set_attributes(0, [-1], [1.0])
    with pytest.raises(N.NativeError):
        store.set_attributes(0, [0], [float("nan")])
    with pytest.raises(N.NativeError):
        store.search_modified(q, 3, [(0, 1.0)] * 17, [])
    with pytest.raises(N.NativeError):
        store.search_modified(q, 3, [(0, float("inf"))], [])
    # attributes of documents beyond the current corpus are accepted (fed before the rows arrive)
    store.set_attributes(0, [500], [2.0])
    doc, _, score = store.search_modified(q, 3, [(0, 10.0)], [])
    assert doc[0, 0] == 0 and abs(score[0, 0] - 1.0) < 1e-6


def test_snapshot_keeps_attributes(gpu_required, score_oracle, tmp_path):
    from marqo_b200.engine import RowStore
    rng = np.random.default_rng(31)
    n, d = 3000, 128
    corpus = K.unit_rows(rng, n, d)
    q = K.unit_rows(rng, 3, d)
    attrs = _attrs(rng, 2, n)
    store = RowStore(d)
    store.add(corpus)
    _feed_attrs(store, attrs)
    path = tmp_path / "snap.b200idx"
    store.save(str(path))
    again = RowStore.load(str(path))
    K.assert_topk_equal(*_search_modified(again, score_oracle, q, corpus, 10, attrs, [(0, 2.0)], [(1, 0.1)]))
