"""GpuTensorIndex fields of any dimension 1 .. 4096 on a CPU stand-in of the row store.

The row store takes widths that are multiples of 64; the adapter stores a d-wide field at round_up(d, 64) with zero
columns appended to every row and query.  The zeros add exact zeros to every product and sum, so nothing a user sees
changes, and the padding never shows: get_batch returns d values and the error messages speak of d."""
import numpy as np
import pytest

import _checks as K
from _filter_scenario import _doc, _yql


class _PaddingStore:
    """RowStore's interface (the part the adapter uses, plus save / load) over numpy: fp16 rows, closeness
    1 / (2 - q.e) in fp64, best chunk per document, (score desc, doc asc).  Keeps every row block it was given."""

    created = []

    def __init__(self, dim, metric="prenormalized-angular", device=0, capacity=0):
        assert dim % 64 == 0 and 0 < dim <= 4096, dim      # what b200_index_create accepts
        self.dim, self.rows, self.docs, self.received = dim, [], [], []
        _PaddingStore.created.append(self)

    def __len__(self):
        return len(self.rows)

    def add(self, vecs, doc_ids=None):
        v = np.asarray(vecs, np.float32)
        assert v.ndim == 2 and v.shape[1] == self.dim, v.shape
        self.received.append(v.copy())
        for i, row in enumerate(v):
            self.rows.append(row.astype(np.float16).astype(np.float64))
            self.docs.append(int(doc_ids[i]) if doc_ids is not None else len(self.docs))

    def delete_rows(self, rows):
        for r in rows:
            self.docs[int(r)] = -1

    def set_attributes(self, column, doc_ids, values):
        pass

    def set_attributes_multi(self, columns, doc_ids, values):
        pass

    def search(self, q, k, mult=(), add=(), filter_bits=None, filter_docs=0, filter_tag=0):
        Q = np.atleast_2d(np.asarray(q, np.float32))
        assert Q.shape[1] == self.dim, Q.shape
        self.received.append(Q.copy())
        out = [np.full((len(Q), k), -1, np.int32), np.full((len(Q), k), -1, np.int32), np.full((len(Q), k), -np.inf)]
        for i, x in enumerate(Q):
            qh = x.astype(np.float16).astype(np.float64)
            best = {}
            for r, (v, d) in enumerate(zip(self.rows, self.docs)):
                if d >= 0:
                    c = 1.0 / (2.0 - float(v @ qh))
                    if d not in best or c > best[d][0]:
                        best[d] = (c, r)
            ranked = sorted(((c, d, r) for d, (c, r) in best.items()), key=lambda t: (-t[0], t[1]))[:k]
            for j, (c, d, r) in enumerate(ranked):
                out[0][i, j], out[1][i, j], out[2][i, j] = d, r, c
        return tuple(out)

    def get_rows(self, rows):
        return np.stack([self.rows[int(r)].astype(np.float32) for r in rows])

    def save(self, path):
        np.savez(path + ".npz", rows=np.asarray(self.rows), docs=np.asarray(self.docs, np.int32))
        with open(path, "w") as fh:
            fh.write(str(self.dim))

    @classmethod
    def load(cls, path, device=0):
        with open(path) as fh:
            st = cls(int(fh.read()))
        z = np.load(path + ".npz")
        st.rows, st.docs = list(z["rows"]), [int(d) for d in z["docs"]]
        return st

    def close(self):
        pass


@pytest.fixture
def gti(monkeypatch):
    import marqo_b200.gpu_tensor_index as gti
    monkeypatch.setattr(gti, "RowStore", _PaddingStore)
    _PaddingStore.created.clear()
    return gti


def _ask(ix, q, hits=5):
    return ix.query(_yql("s1", ["body"], hits), hits=hits, ranking="embedding_similarity", model_restrict="s1",
                    query_features={"marqo__query_embedding": np.asarray(q).tolist()})


def _expected(vecs, chunks, q, hits):
    """(document index, closeness) of the best `hits` documents, from the unpadded vectors."""
    qh = q.astype(np.float16).astype(np.float64)
    c = 1.0 / (2.0 - vecs.astype(np.float16).astype(np.float64) @ qh)
    best = c.reshape(-1, chunks).max(axis=1)
    order = sorted(range(len(best)), key=lambda i: (-best[i], i))[:hits]
    return [f"d{i}" for i in order], [float(best[i]) for i in order]


@pytest.mark.parametrize("d", [16, 32, 100, 234, 1000])
def test_any_dimension_feeds_queries_reads_back_and_persists(gti, d, tmp_path):
    rng = np.random.default_rng(d)
    n, chunks = 30, 2
    vecs = K.unit_rows(rng, n * chunks, d)
    ix = gti.GpuTensorIndex()
    docs = [_doc(f"d{i}", {}, {"body": (["c0", "c1"], vecs[i * chunks:(i + 1) * chunks])}) for i in range(n)]
    assert not ix.feed_batch(docs, "s1").errors
    (store,) = _PaddingStore.created
    width = -(-d // 64) * 64
    assert store.dim == width
    # every row the store received carries exact zeros beyond column d
    for block in store.received:
        assert block.shape[1] == width and not block[:, d:].any()
    np.testing.assert_array_equal(np.concatenate(store.received)[:, :d], vecs)
    q = K.unit_rows(rng, 1, d)[0]
    res = _ask(ix, q)
    ids, rel = _expected(vecs, chunks, q, 5)
    assert [h.id.split("::")[-1] for h in res.hits] == ids
    assert [h.relevance for h in res.hits] == rel
    assert store.received[-1].shape == (1, width) and not store.received[-1][:, d:].any()
    # get_batch: d values per chunk, the fp16 values that were stored
    got = ix.get_batch(["d3"], "s1").responses[0].document.fields["marqo__embeddings_body"]
    assert sorted(got) == ["0", "1"] and all(len(v) == d for v in got.values())
    np.testing.assert_array_equal(np.asarray(got["1"], np.float32), vecs[7].astype(np.float16).astype(np.float32))
    # save / load keeps d
    ix.save(str(tmp_path))
    back = gti.GpuTensorIndex.load(str(tmp_path))
    res2 = _ask(back, q)
    assert [h.id for h in res2.hits] == [h.id for h in res.hits]
    got2 = back.get_batch(["d3"], "s1").responses[0].document.fields["marqo__embeddings_body"]
    assert got2 == got
    with pytest.raises(Exception, match=f"dimension {d} for query input but got {d + 1}"):
        _ask(back, np.zeros(d + 1, np.float32))


@pytest.mark.parametrize("d", [16, 234])
def test_wrong_dimension_documents_and_queries_are_rejected(gti, d):
    rng = np.random.default_rng(1)
    ix = gti.GpuTensorIndex()
    assert not ix.feed_batch([_doc("a", {}, {"body": (["0"], K.unit_rows(rng, 1, d))})], "s1").errors
    for bad in (d - 1, d + 1, -(-d // 64) * 64):      # the padded width is not the field's dimension either
        r = ix.feed_batch([_doc("b", {}, {"body": (["0"], K.unit_rows(rng, 1, bad))})], "s1")
        assert r.errors and r.responses[0].status == 400
        assert r.responses[0].message == f"field marqo__embeddings_body: embedding dimension {bad} != index dimension {d}"
        with pytest.raises(Exception, match=f"Expected a tensor of dimension {d} for query input but got {bad}"):
            _ask(ix, np.zeros(bad, np.float32))
    assert ix.get_document_count("s1") == 1


def test_device_chunks_on_a_padded_field_are_rejected(gti):
    ix = gti.GpuTensorIndex()
    r = ix.feed_batch([{"id": "a", "fields": {"marqo__embeddings_body": gti.DeviceChunks(["0"], 0, 100)}}], "s1")
    assert r.errors and r.responses[0].status == 400
    assert "not a multiple of 64" in r.responses[0].message
    assert not _PaddingStore.created


@pytest.mark.parametrize("d", [4097, 6144])
def test_dimensions_above_4096_are_rejected(gti, d):
    ix = gti.GpuTensorIndex()
    mat = {"0": [0.5] * d}
    r = ix.feed_batch([{"id": "a", "fields": {"marqo__embeddings_body": mat}}], "s1")
    assert r.errors and r.responses[0].status == 400
    assert r.responses[0].message == f"field marqo__embeddings_body: embedding dimension {d} is not in [1, 4096]"
    assert not _PaddingStore.created


def test_manifest_without_a_recorded_dimension_loads_at_the_store_width(gti, tmp_path):
    """Snapshots written before fields could be padded have no "dim" entry: the field's dimension is the store's."""
    import json
    rng = np.random.default_rng(2)
    vecs = K.unit_rows(rng, 4, 128)
    ix = gti.GpuTensorIndex()
    ix.feed_batch([_doc(f"d{i}", {}, {"body": (["0"], vecs[i:i + 1])}) for i in range(4)], "s1")
    ix.save(str(tmp_path))
    manifest = json.loads((tmp_path / "manifest.json").read_text())
    assert "dim" not in manifest["schemas"]["s1"]["stores"]["marqo__embeddings_body"]
    back = gti.GpuTensorIndex.load(str(tmp_path))
    got = back.get_batch(["d1"], "s1").responses[0].document.fields["marqo__embeddings_body"]
    assert len(got["0"]) == 128
    assert [h.id.split("::")[-1] for h in _ask(back, vecs[2], hits=1).hits] == ["d2"]
