"""GPU parity tests for the score + top-k path (SURVEY §8 a8) — CUDA path through the C ABI vs oracle/score_oracle.c.

Bar: doc ids and arg-max rows bit-exact; closeness equal to 1e-12 (fp64; acos may differ in the last ulp).
"""
import numpy as np
import pytest

import _checks as K

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n,d,nq,k", [
    (1, 64, 1, 1), (7, 64, 3, 10), (128, 128, 64, 10), (129, 256, 5, 3), (1000, 768, 64, 10),
    (20000, 768, 64, 10), (33333, 512, 17, 16), (5000, 1024, 64, 10), (4097, 384, 100, 10),
])
def test_topk_matches_oracle(gpu_required, score_oracle, n, d, nq, k):
    from marqo_b200.engine import RowStore
    rng = np.random.default_rng(n * 31 + d)
    corpus = K.unit_rows(rng, n, d)
    q = K.unit_rows(rng, nq, d)
    store = RowStore(d)
    store.add(corpus)
    assert len(store) == n
    K.assert_topk_equal(store.search(q, k), score_oracle.search(q, corpus, k, "prenormalized-angular"))


def test_self_match_and_duplicates(gpu_required, score_oracle):
    """SURVEY §8(d) cfg5: queries copied from corpus rows rank first with closeness ~ 1; duplicated rows tie and
    are returned in ascending doc order (the defined tie rule)."""
    from marqo_b200.engine import RowStore
    rng = np.random.default_rng(5)
    n, d = 30000, 768
    corpus = K.unit_rows(rng, n, d)
    corpus[20000:20050] = corpus[123]          # 50 exact duplicates of row 123
    corpus[777] = corpus[29999]
    q = K.unit_rows(rng, 64, d)
    q[:8] = corpus[[123, 5, 999, 15000, 29999, 4242, 64, 127]]
    store = RowStore(d)
    store.add(corpus)
    doc, row, score = store.search(q, 10)
    assert doc[0, 0] == 123 and list(doc[0, 1:10]) == list(range(20000, 20009))
    assert doc[4, 0] == 777 and doc[4, 1] == 29999
    assert np.all(np.abs(score[:8, 0] - 1.0) < 2e-3)
    K.assert_topk_equal(store.search(q, 10), score_oracle.search(q, corpus, 10, "prenormalized-angular"))


@pytest.mark.parametrize("metric", ["angular", "dotproduct", "euclidean"])
def test_other_metrics(gpu_required, score_oracle, metric):
    from marqo_b200.engine import RowStore
    rng = np.random.default_rng(9)
    corpus = rng.standard_normal((3000, 256)).astype(np.float32)
    q = rng.standard_normal((9, 256)).astype(np.float32)
    store = RowStore(256, metric=metric)
    store.add(corpus[:1000])
    store.add(corpus[1000:])
    K.assert_topk_equal(store.search(q, 10), score_oracle.search(q, corpus, 10, metric))
    doc_of_row = (np.arange(3000) // 2).astype(np.int32)
    chunks = RowStore(256, metric=metric)
    chunks.add(corpus, doc_of_row)
    K.assert_topk_equal(chunks.search(q, 25), score_oracle.search(q, corpus, 25, metric, doc_of_row))
    if metric == "euclidean":
        d, r, s = store.search(corpus[5:6], 1)
        # distance to its own fp16-rounded copy is tiny but not 0 (query is rounded too -> identical -> exactly 0)
        assert d[0, 0] == 5 and s[0, 0] == 1.0


def test_max_over_chunks_and_delete(gpu_required, score_oracle):
    """score(doc) = max over chunks (unstructured_vespa_schema.py:225-230); deleted docs never surface."""
    from marqo_b200.engine import RowStore
    rng = np.random.default_rng(11)
    n, d = 9000, 256
    corpus = K.unit_rows(rng, n, d)
    doc_of_row = (np.arange(n) // 3).astype(np.int32)            # 3 chunks per doc
    doc_of_row[6000:] = rng.integers(0, 3000, size=3000)          # plus scattered extra chunks
    q = K.unit_rows(rng, 40, d)
    q[0] = corpus[4]                                              # doc 1, chunk row 4
    store = RowStore(d)
    store.add(corpus[:5000], doc_of_row[:5000])
    store.add(corpus[5000:], doc_of_row[5000:])
    doc, row, score = store.search(q, 10)
    assert doc[0, 0] == 1 and row[0, 0] == 4
    for qi in range(doc.shape[0]):
        assert len(set(doc[qi])) == 10                            # one hit per document
    K.assert_topk_equal(store.search(q, 10), score_oracle.search(q, corpus, 10, "prenormalized-angular", doc_of_row))
    store.delete_doc(1)
    dd = doc_of_row.copy()
    dd[dd == 1] = -1
    doc2, _, _ = store.search(q, 10)
    assert 1 not in doc2[0]
    K.assert_topk_equal(store.search(q, 10), score_oracle.search(q, corpus, 10, "prenormalized-angular", dd))


@pytest.mark.parametrize("k", [11, 16, 50, 200])
def test_large_k_multi_round(gpu_required, score_oracle, k):
    """k beyond the single-pass limit (Marqo allows limit <= 1000): multi-round scan, same exact order."""
    from marqo_b200.engine import RowStore
    rng = np.random.default_rng(k)
    n, d = 6000, 128
    corpus = K.unit_rows(rng, n, d)
    corpus[100:140] = corpus[5]                                   # a run of exact ties across the round boundary
    doc_of_row = (np.arange(n) // 2).astype(np.int32)            # 2 chunks per doc
    q = K.unit_rows(rng, 7, d)
    q[0] = corpus[5]
    store = RowStore(d)
    store.add(corpus, doc_of_row)
    K.assert_topk_equal(store.search(q, k), score_oracle.search(q, corpus, k, "prenormalized-angular", doc_of_row))
    small = RowStore(d)
    small.add(corpus[:30])                                        # fewer documents than k
    doc, row, score = small.search(q[:2], k)
    assert (doc[:, :30] >= 0).all() and (doc[:, 30:] == -1).all()
    K.assert_topk_equal(small.search(q[:2], k), score_oracle.search(q[:2], corpus[:30], k, "prenormalized-angular"))


def test_empty_and_small(gpu_required):
    from marqo_b200.engine import RowStore
    store = RowStore(64)
    doc, row, score = store.search(np.ones((2, 64), np.float32), 5)
    assert (doc == -1).all() and (row == -1).all() and np.isneginf(score).all()
    store.add(np.eye(3, 64, dtype=np.float32))
    doc, row, score = store.search(np.eye(1, 64, dtype=np.float32), 5)
    assert list(doc[0]) == [0, 1, 2, -1, -1]
    assert score[0, 0] == 1.0                                    # identical vector => _score == 1.0
    assert score[0, 1] == 0.5 and np.isneginf(score[0, 3])


def test_growth_and_snapshot(gpu_required, score_oracle, tmp_path):
    from marqo_b200.engine import RowStore
    rng = np.random.default_rng(3)
    d = 128
    corpus = K.unit_rows(rng, 2500, d)
    store = RowStore(d, capacity=10)
    for lo in range(0, 2500, 700):
        store.add(corpus[lo:lo + 700])
    q = K.unit_rows(rng, 6, d)
    K.assert_topk_equal(store.search(q, 10), score_oracle.search(q, corpus, 10, "prenormalized-angular"))
    np.testing.assert_array_equal(store.get_row(17), corpus[17].astype(np.float16).astype(np.float32))
    p = tmp_path / "snap.b200"
    store.save(str(p))
    again = RowStore.load(str(p))
    assert len(again) == 2500 and again.dim == d
    K.assert_topk_equal(again.search(q, 10), score_oracle.search(q, corpus, 10, "prenormalized-angular"))


def test_argument_errors(gpu_required):
    from marqo_b200.engine import RowStore
    from marqo_b200._native import NativeError
    with pytest.raises(NativeError):
        RowStore(100)                                            # dim not a multiple of 64
    store = RowStore(64)
    with pytest.raises(ValueError):
        store.add(np.zeros((2, 32), np.float32))
    with pytest.raises(NativeError):
        store.search(np.zeros((1, 64), np.float32), 0)


def test_doc_offset_and_device_shard_merge(gpu_required, score_oracle):
    """Row-sharded search on one GPU: two stores with document offsets, packed result blocks, device-side merge ==
    oracle top-k over the concatenated corpus (the N > 1 data path minus the NCCL transport)."""
    import torch
    from marqo_b200.engine import RowStore
    rng = np.random.default_rng(21)
    n, d, nq, k = 5000, 128, 33, 10
    corpus = K.unit_rows(rng, n, d)
    corpus[4000] = corpus[10]                                   # cross-shard tie: lower doc id first
    q = K.unit_rows(rng, nq, d)
    q[0] = corpus[10]
    cut = 2300
    shards = [RowStore(d), RowStore(d)]
    shards[0].add(corpus[:cut])
    shards[1].add(corpus[cut:])
    shards[1].set_doc_offset(cut)
    nk = nq * k
    qd = torch.from_numpy(q).cuda()
    gathered = torch.empty(2 * nk * 16, dtype=torch.uint8, device="cuda")
    for i, st in enumerate(shards):
        base = gathered.data_ptr() + i * nk * 16
        st.search_device(qd.data_ptr(), nq, k, base, base + nk * 4, base + nk * 8, sync=True)
    od = torch.empty(nq, k, dtype=torch.int32, device="cuda")
    orow = torch.empty_like(od)
    osc = torch.empty(nq, k, dtype=torch.float64, device="cuda")
    shards[0].merge_shards_device(gathered.data_ptr(), 2, nq, k, od.data_ptr(), orow.data_ptr(), osc.data_ptr())
    ed, er, es = score_oracle.search(q, corpus, k)
    np.testing.assert_array_equal(od.cpu().numpy(), ed)
    np.testing.assert_allclose(osc.cpu().numpy(), es, rtol=0, atol=1e-12)
    assert od[0, 0].item() == 10 and od[0, 1].item() == 4000
    # rows are shard-local (they index the shard's matrix): check through the doc numbers
    lr = orow.cpu().numpy()
    assert ((lr == ed) | (lr == ed - cut)).all()
