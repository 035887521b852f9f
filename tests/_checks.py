"""Checks and inputs shared by the test files: embedding parity against an oracle, top-k parity against the score
oracle, and the vectorise -> GpuTensorIndex -> search seam, each written once so that every model family is held to the
same bar."""
import numpy as np
import torch

COS_TOL = 1e-3   # BASELINE.json north_star: cosine >= 1 - 1e-3 per vector


def bf16(x: torch.Tensor) -> torch.Tensor:
    """Round to bf16 (round to nearest even) and back to fp32."""
    return x.to(torch.bfloat16).to(torch.float32)


def _cpu(x) -> torch.Tensor:
    """A numpy array, a nested list, or a CPU or CUDA tensor as a CPU tensor."""
    return x.cpu() if isinstance(x, torch.Tensor) else torch.as_tensor(np.asarray(x))


def cosine(a, b) -> torch.Tensor:
    """Row-wise cosine similarity of a and b, in fp64."""
    return torch.nn.functional.cosine_similarity(_cpu(a).double(), _cpu(b).double(), dim=-1)


def assert_embeddings_match(got, ref, tol=COS_TOL, unit_norm=True):
    """Every row of got is finite and has a cosine above 1 - tol with the same row of ref; with unit_norm, every row of
    got also has a norm within 1e-5 of 1."""
    got = _cpu(got)
    assert torch.isfinite(got).all()
    c = cosine(got, ref)
    assert float((1 - c).max()) < tol, f"min cosine {float(c.min())}"
    if unit_norm:
        assert torch.allclose(got.norm(dim=-1), torch.ones(got.shape[0], dtype=got.dtype), atol=1e-5)


def assert_topk_equal(got, expected, atol=1e-12):
    """Two (doc, row, score) top-k results: ids and rows equal, scores within atol.  Returns got."""
    doc, row, score = got
    edoc, erow, escore = expected
    np.testing.assert_array_equal(doc, edoc)
    np.testing.assert_array_equal(row, erow)
    np.testing.assert_allclose(score, escore, rtol=0, atol=atol)
    return got


def assert_index_search_matches(score_oracle, docs, queries, k=10):
    """Feed docs [n, D] to a GpuTensorIndex under schema s1, one chunk per document with ids d0, d1, ..., and run an
    exact nearestNeighbor search for each row of queries: the hit ids are the score oracle's prenormalized-angular top
    k and the relevances its scores within 1e-12."""
    from marqo_b200.gpu_tensor_index import GpuTensorIndex
    ix = GpuTensorIndex()
    feed = [{"id": f"d{i}", "fields": {"marqo__id": f"d{i}", "marqo__chunks_body": ["c"],
                                       "marqo__embeddings_body": {"0": v.tolist()}}} for i, v in enumerate(docs)]
    assert not ix.feed_batch(feed, "s1").errors
    yql = (f"select * from s1 where (({{targetHits:{k}, approximate:False, hnsw.exploreAdditionalHits:0}}"
           f"nearestNeighbor(marqo__embeddings_body, marqo__query_embedding)))")
    edoc, _, escore = score_oracle.search(queries, docs, k, "prenormalized-angular")
    for j in range(len(queries)):
        res = ix.query(yql, hits=k, ranking="embedding_similarity", model_restrict="s1",
                       query_features={"marqo__query_embedding": queries[j].tolist()})
        assert [h.id.split("::")[-1] for h in res.hits] == [f"d{d}" for d in edoc[j]]
        np.testing.assert_allclose([h.relevance for h in res.hits], escore[j], rtol=0, atol=1e-12)
    ix.close()


def unit_rows(rng, n, d):
    """n random fp32 rows of dimension d, each of norm 1."""
    x = rng.standard_normal((n, d)).astype(np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    return x


def sample_positions(n, m):
    """Up to m positions spread over a batch of n, the first and the last among them, in ascending order."""
    return sorted(set([0, n - 1] + [int(x) for x in np.linspace(1, n - 2, m - 2)]))


class WordTokenizer:
    """Stand-in for AutoTokenizer (no vocab files offline): 'w<i>' words -> ids offset + i, between cls_id and sep_id,
    padded with 0."""

    def __init__(self, cls_id, sep_id, offset):
        self.cls_id, self.sep_id, self.offset = cls_id, sep_id, offset

    def __call__(self, sentences, padding=True, truncation=True, max_length=128, return_tensors="np"):
        rows = [[self.cls_id] + [self.offset + int(w[1:]) for w in s.split()][: max_length - 2] + [self.sep_id]
                for s in sentences]
        L = max(len(r) for r in rows)
        ids = np.zeros((len(rows), L), np.int64)
        mask = np.zeros((len(rows), L), np.int64)
        for i, r in enumerate(rows):
            ids[i, :len(r)] = r
            mask[i, :len(r)] = 1
        return {"input_ids": ids, "attention_mask": mask}
