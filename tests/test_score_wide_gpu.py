"""Row stores wider than 1024 (score.cu: the streamed-query scan kernel) and the adapter's zero-padded fields of any
dimension, checked bit for bit against oracle/score_oracle.c.

Above dim 1024 the query block no longer fits in shared memory beside the ring stages, so every ring stage carries
the query k-block next to the corpus k-block.  b200_debug_index_scan_kernel reports which kernel a search ran and can
force the streamed kernel at any dim, so both kernels are run on one corpus here; every case asserts the kernel."""
import numpy as np
import pytest

import _checks as K

pytestmark = pytest.mark.gpu

WIDE_DIMS = [1088, 1152, 1536, 2048, 3072, 4096]
METRICS = ["prenormalized-angular", "angular", "dotproduct", "euclidean"]


def _rows_for(metric, rng, n, d):
    if metric in ("prenormalized-angular", "angular"):
        return K.unit_rows(rng, n, d)
    return K.unit_rows(rng, n, d) * np.float32(0.7)     # not unit: the dot product and distance use the norms


def _expect(so, q, corpus, k, metric="prenormalized-angular", doc_of_row=None, got=None):
    edoc, erow, escore = so.search(q, corpus, k, metric, doc_of_row)
    doc, row, score = got
    np.testing.assert_array_equal(doc, edoc)
    np.testing.assert_array_equal(row, erow)
    _same_scores(score, escore, metric)


def _same_scores(score, escore, metric="prenormalized-angular"):
    """Bitwise, except that the angular closeness goes through acos: CUDA's double acos is within 2 ulp and the host C
    library's within 1, so the two closeness values may differ by a few ulp (the dot products under them, and with
    them the ids and rows, are bitwise equal)."""
    if metric != "angular":
        np.testing.assert_array_equal(score, escore)
        return
    fin = np.isfinite(escore)
    np.testing.assert_array_equal(np.isfinite(score), fin)
    np.testing.assert_array_max_ulp(score[fin], escore[fin], maxulp=4)


def _kernel(store):
    from marqo_b200.engine import debug_scan_kernel
    return debug_scan_kernel(store)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("d", WIDE_DIMS)
def test_wide_rows_match_the_oracle(gpu_required, score_oracle, d, metric):
    """Multi-chunk documents with a permuted row -> document map, tombstones, k from 1 to 1000."""
    from marqo_b200 import _native as N
    from marqo_b200.engine import RowStore
    rng = np.random.default_rng(d + len(metric))
    n = 24_000_000 // d                       # 5.8 k .. 22 k rows
    corpus = _rows_for(metric, rng, n, d)
    corpus[40:60] = corpus[3]                                     # exact duplicates
    doc_of_row = (rng.permutation(n) // 3).astype(np.int32)       # 3 chunks per document, scattered over the matrix
    q = _rows_for(metric, rng, 6, d)
    q[0] = corpus[3]
    store = RowStore(d, metric=metric)
    assert _kernel(store) == -1
    store.add(corpus, doc_of_row)
    dead = rng.choice(n, size=n // 10, replace=False)
    store.delete_rows(dead)
    masked = doc_of_row.copy()
    masked[dead] = -1
    for k in (1, 10, 160, 1000):
        _expect(score_oracle, q, corpus, k, metric, masked, store.search(q, k))
        assert _kernel(store) == N.SCAN_STREAMED_Q


def test_many_tiles_per_sm(gpu_required, score_oracle):
    """200 k rows of 1536: about twelve 128-row tiles per SM, so the ring wraps many times per CTA."""
    from marqo_b200 import _native as N
    from marqo_b200.engine import RowStore
    rng = np.random.default_rng(11)
    n, d = 200_000, 1536
    corpus = K.unit_rows(rng, n, d)
    q = K.unit_rows(rng, 8, d)
    q[0] = corpus[n - 1]
    store = RowStore(d)
    store.add(corpus)
    _expect(score_oracle, q, corpus, 10, got=store.search(q, 10))
    assert _kernel(store) == N.SCAN_STREAMED_Q


def test_filter_and_modifiers_1536(gpu_required, score_oracle):
    from marqo_b200 import _native as N
    from marqo_b200.engine import RowStore
    rng = np.random.default_rng(12)
    n, d = 16_000, 1536
    corpus = K.unit_rows(rng, n, d)
    doc_of_row = (np.arange(n) // 2).astype(np.int32)
    ndocs = n // 2
    q = K.unit_rows(rng, 5, d)
    store = RowStore(d)
    store.add(corpus, doc_of_row)
    keep = rng.random(ndocs) < 0.2
    bits = np.packbits(keep, bitorder="little")
    bits = np.concatenate([bits, np.zeros((-len(bits)) % 4, np.uint8)]).view(np.uint32)
    masked = np.where(keep[doc_of_row], doc_of_row, -1).astype(np.int32)
    for k in (10, 200):
        got = store.search(q, k, filter_bits=bits, filter_docs=ndocs)
        assert _kernel(store) == N.SCAN_STREAMED_Q
        _expect(score_oracle, q, corpus, k, doc_of_row=masked, got=got)
    vals = rng.uniform(0.5, 2.0, size=ndocs)
    store.set_attributes_multi(np.zeros(ndocs, np.int32), np.arange(ndocs, dtype=np.int32), vals)
    mod = score_oracle.modifiers(vals[None, :], [(0, 1.5)], [(0, 0.01)])
    doc, row, score = store.search(q, 10, mult=[(0, 1.5)], add=[(0, 0.01)])
    assert _kernel(store) == N.SCAN_STREAMED_Q
    ed, er, es = score_oracle.search_modified(q, corpus, 10, mod, doc_of_row=doc_of_row)
    np.testing.assert_array_equal(doc, ed)
    np.testing.assert_array_equal(row, er)
    np.testing.assert_array_equal(score, es)


def test_ties_and_near_ties_3072(gpu_required, score_oracle):
    """100 identical rows and a family of rows within 1e-7 of each other around rank k: the guard must flag the
    query and the collect pass answer it."""
    from marqo_b200 import _native as N
    from marqo_b200.engine import RowStore
    rng = np.random.default_rng(13)
    n, d = 60_000, 3072
    corpus = K.unit_rows(rng, n, d)
    # 20 identical rows in one tile (more than one CTA's 16-entry list holds) and 80 more elsewhere (more than the 64
    # candidates the merge re-scores for k <= 10)
    ties = np.concatenate([np.arange(2000, 2020), rng.choice(np.arange(3000, n), size=80, replace=False)])
    corpus[ties] = corpus[ties[0]]
    base = corpus[77].copy()
    h = base.astype(np.float16)
    small = np.argsort(np.abs(h.astype(np.float32)))[8:8 + 64]
    fam = np.repeat(h[None, :], 30, axis=0)
    for i in range(30):                                          # one-ulp moves of small components: ~1e-9 apart
        bits = fam[i].view(np.uint16).copy()
        bits[rng.choice(small, size=1 + i % 3, replace=False)] += np.uint16(1 + i % 2)
        fam[i] = bits.view(np.float16)
    near = rng.choice(np.setdiff1d(np.arange(n), ties), size=30, replace=False)
    corpus[near] = fam.astype(np.float32)
    q = K.unit_rows(rng, 4, d)
    q[0] = corpus[ties[0]]
    q[1] = base
    store = RowStore(d)
    store.add(corpus)
    for k in (10, 25, 120):
        _expect(score_oracle, q, corpus, k, got=store.search(q, k))
        assert _kernel(store) == N.SCAN_STREAMED_Q
    st = store.search_stats()
    assert st["flagged"] > 0 and st["collect_passes"] > 0, st


def test_async_compact_save_load_rows_and_device_merge_1536(gpu_required, score_oracle, tmp_path):
    import torch
    from marqo_b200 import _native as N
    from marqo_b200.engine import RowStore
    rng = np.random.default_rng(14)
    n, d, nq, k = 12_000, 1536, 6, 10
    corpus = K.unit_rows(rng, n, d)
    corpus[500:530] = corpus[9]
    q = K.unit_rows(rng, nq, d)
    q[0] = corpus[9]
    store = RowStore(d)
    store.add(corpus)
    # asynchronous device entry point: the fallback pass runs without the host
    qd = torch.from_numpy(q).cuda()
    od = torch.empty(nq, k, dtype=torch.int32, device="cuda")
    orow = torch.empty_like(od)
    osc = torch.empty(nq, k, dtype=torch.float64, device="cuda")
    store.search_device(qd.data_ptr(), nq, k, od.data_ptr(), orow.data_ptr(), osc.data_ptr(), sync=False)
    torch.cuda.synchronize()
    assert _kernel(store) == N.SCAN_STREAMED_Q
    _expect(score_oracle, q, corpus, k, got=(od.cpu().numpy(), orow.cpu().numpy(), osc.cpu().numpy()))
    assert store.search_stats()["unresolved_async"] == 0
    # get_rows gives the fp16-rounded rows back
    rows = np.array([0, 9, 511, n - 1])
    np.testing.assert_array_equal(store.get_rows(rows), corpus[rows].astype(np.float16).astype(np.float32))
    # tombstones + compaction
    dead = rng.choice(n, size=4000, replace=False)
    store.delete_rows(dead)
    new_of_old = store.compact()
    live = np.flatnonzero(new_of_old >= 0)
    assert len(live) == n - 4000
    _expect(score_oracle, q, corpus[live], k, doc_of_row=live.astype(np.int32), got=store.search(q, k))
    # snapshot round trip
    path = str(tmp_path / "wide.b200idx")
    store.save(path)
    back = RowStore.load(path)
    assert back.dim == d
    _expect(score_oracle, q, corpus[live], k, doc_of_row=live.astype(np.int32), got=back.search(q, k))
    assert _kernel(back) == N.SCAN_STREAMED_Q
    # two row shards with a document offset, merged on the device
    cut = 7000
    shards = [RowStore(d), RowStore(d)]
    shards[0].add(corpus[:cut])
    shards[1].add(corpus[cut:])
    shards[1].set_doc_offset(cut)
    nk = nq * k
    gathered = torch.empty(2 * nk * 16, dtype=torch.uint8, device="cuda")
    for i, st in enumerate(shards):
        b = gathered.data_ptr() + i * nk * 16
        st.search_device(qd.data_ptr(), nq, k, b, b + nk * 4, b + nk * 8, sync=True)
    shards[0].merge_shards_device(gathered.data_ptr(), 2, nq, k, od.data_ptr(), orow.data_ptr(), osc.data_ptr())
    ed, _, es = score_oracle.search(q, corpus, k)
    np.testing.assert_array_equal(od.cpu().numpy(), ed)
    np.testing.assert_array_equal(osc.cpu().numpy(), es)


@pytest.mark.parametrize("metric", ["prenormalized-angular", "euclidean"])
@pytest.mark.parametrize("d", [64, 768, 1024])
def test_forced_streamed_kernel_equals_resident(gpu_required, score_oracle, d, metric):
    """The same corpus through both kernels: identical ids, rows and scores, and both equal to the oracle."""
    from marqo_b200 import _native as N
    from marqo_b200.engine import RowStore, debug_scan_kernel
    rng = np.random.default_rng(d)
    n = 30_000
    corpus = _rows_for(metric, rng, n, d)
    corpus[100:130] = corpus[5]
    doc_of_row = (np.arange(n) // 2).astype(np.int32)
    q = _rows_for(metric, rng, 7, d)
    q[0] = corpus[5]
    store = RowStore(d, metric=metric)
    store.add(corpus, doc_of_row)
    for k in (10, 1000):
        resident = store.search(q, k)
        assert debug_scan_kernel(store) == N.SCAN_RESIDENT_Q
        assert debug_scan_kernel(store, force_streamed=True) == N.SCAN_RESIDENT_Q   # reports the last search
        streamed = store.search(q, k)
        assert debug_scan_kernel(store, force_streamed=False) == N.SCAN_STREAMED_Q
        for a, b in zip(resident, streamed):
            np.testing.assert_array_equal(a, b)
        _expect(score_oracle, q, corpus, k, metric, doc_of_row, streamed)


def test_dim_above_4096_is_rejected(gpu_required):
    from marqo_b200 import _native as N
    from marqo_b200.engine import RowStore
    with pytest.raises(N.NativeError) as e:
        RowStore(4160)
    assert e.value.code == N.ERR_INVALID_ARG
    RowStore(4096).close()


@pytest.mark.parametrize("d", [16, 234])
def test_adapter_pads_narrow_fields(gpu_required, score_oracle, d, tmp_path):
    """GpuTensorIndex stores a d-wide field at round_up(d, 64) with zero columns: the results are those of the
    unpadded vectors, and get_batch gives back d values."""
    from _filter_scenario import _doc, _yql
    from marqo_b200.gpu_tensor_index import GpuTensorIndex
    rng = np.random.default_rng(d)
    n_docs, chunks = 400, 2
    vecs = K.unit_rows(rng, n_docs * chunks, d)
    ix = GpuTensorIndex()
    docs = [_doc(f"d{i}", {}, {"body": ([f"c{j}" for j in range(chunks)], vecs[i * chunks:(i + 1) * chunks])})
            for i in range(n_docs)]
    resp = ix.feed_batch(docs, "s1")
    assert not resp.errors
    q = K.unit_rows(rng, 3, d)
    doc_of_row = (np.arange(n_docs * chunks) // chunks).astype(np.int32)
    w = -(-d // 64) * 64                      # the oracle's summation order needs a multiple of 8: pad as the adapter does
    pad = lambda x: np.concatenate([x, np.zeros((x.shape[0], w - d), np.float32)], axis=1)
    ed, _, es = score_oracle.search(pad(q), pad(vecs), 10, doc_of_row=doc_of_row)

    def ask(index, qv):
        res = index.query(_yql("s1", ["body"], 10), hits=10, ranking="embedding_similarity", model_restrict="s1",
                          query_features={"marqo__query_embedding": qv.tolist()})
        return [h.id.split("::")[-1] for h in res.hits], [h.relevance for h in res.hits]

    for i in range(3):
        ids, rel = ask(ix, q[i])
        assert ids == [f"d{x}" for x in ed[i]]
        assert rel == list(es[i])
    got = ix.get_batch(["d7"], "s1").responses[0].document.fields["marqo__embeddings_body"]
    assert sorted(got) == ["0", "1"] and len(got["0"]) == d
    np.testing.assert_array_equal(np.asarray(got["1"], np.float32), vecs[15].astype(np.float16).astype(np.float32))
    ix.save(str(tmp_path))
    back = GpuTensorIndex.load(str(tmp_path))
    ids, rel = ask(back, q[0])
    assert ids == [f"d{x}" for x in ed[0]] and rel == list(es[0])
