"""Checks and inputs shared by the test files: embedding parity against an oracle, every input path of an image tower,
refusals at create time, top-k parity against the score oracle, and the vectorise -> GpuTensorIndex -> search seam,
each written once so that every model family is held to the same bar.  A file whose torch oracle runs on the GPU
imports the autouse fixture fp32_oracle by name."""
import numpy as np
import pytest
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


@pytest.fixture(autouse=True)
def fp32_oracle():
    """TF32 off for torch's matmuls and cuDNN convolutions while a test runs, so that a GPU oracle computes in fp32."""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _assert_rows_match(got, ref, unit_norm):
    """assert_embeddings_match, and every row's norm within 1 % of ref's, so that normalised and unnormalised rows
    cannot stand in for each other."""
    assert_embeddings_match(got, ref, unit_norm=unit_norm)
    torch.testing.assert_close(_cpu(got).double().norm(dim=-1), _cpu(ref).double().norm(dim=-1), rtol=1e-2, atol=0)


def check_image_input_paths(enc, at_size, photo, preprocess, ref, rows=None, resize=None):
    """Encoder enc's image tower on every input path against ref(chw, normalize), the oracle on preprocess(u8), fp32
    [n, 3, S, S]:

      - uint8 images at the model's size, the given rows of them (all by default) against ref;
      - the same images from device memory: the same bits;
      - photo (uint8 of another size) through the model's resize; with resize (that resize kernel alone), also the bits
        of photo resized by it first;
      - photo's first three rows preprocessed to fp32;
      - unnormalised rows from the uint8 and the fp32 path.

    Returns the embeddings of at_size."""
    n, S = len(at_size), enc.image_size
    rows = list(range(n)) if rows is None else rows
    got = enc.encode_images_u8(at_size)
    assert got.shape == (n, enc.embed_dim)
    _assert_rows_match(got[rows], ref(preprocess(at_size[rows]), normalize=True), True)
    d_in = torch.from_numpy(at_size).cuda()
    out = torch.empty((n, enc.embed_dim), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    enc.encode_images_u8_device(d_in.data_ptr(), n, S, S, out.data_ptr(), sync=True)
    np.testing.assert_array_equal(out.cpu().numpy(), got)
    resized = enc.encode_images_u8(photo)
    _assert_rows_match(resized, ref(preprocess(photo), normalize=True), True)
    if resize is not None:
        np.testing.assert_array_equal(resized, enc.encode_images_u8(resize(photo, S)))
    chw = preprocess(photo[:3])
    _assert_rows_match(enc.encode_images_f32(chw.numpy()), ref(chw, normalize=True), True)
    raw = enc.encode_images_u8(at_size[:2], normalize=False)
    _assert_rows_match(raw, ref(preprocess(at_size[:2]), normalize=False), False)
    _assert_rows_match(enc.encode_images_f32(chw.numpy(), normalize=False), ref(chw, normalize=False), False)
    return got


def clip_text_ids(n, seed):
    """n CLIP token rows of 77: start 49406, 1 to 68 random ids, end 49407, zero padding."""
    ids = torch.zeros(n, 77, dtype=torch.int64)
    g = torch.Generator().manual_seed(seed)
    for i in range(n):
        L = int(torch.randint(2, 70, (1,), generator=g))
        ids[i, 0] = 49406
        ids[i, 1:L] = torch.randint(1, 49000, (L - 1,), generator=g)
        ids[i, L] = 49407
    return ids


def assert_refused(kind, arch, weights, code, in_message=None):
    """Encoder(kind, arch, weights) is refused with NativeError code, whose message names in_message if given."""
    from marqo_b200._native import NativeError
    from marqo_b200.engine import Encoder
    with pytest.raises(NativeError) as e:
        Encoder(kind, arch, weights, max_batch=2)
    assert e.value.code == code, e.value
    assert in_message is None or in_message in e.value.message, e.value


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


def served_resize_sizes(mode):
    """The image sizes S that the served image towers resize to in `mode`: "crop" (the shortest side to S, then the
    centre S x S) or "squash" (both sides to S), as each entry's arch.get("resize_mode") says (crop by default)."""
    from marqo_b200 import model_registry as R
    sizes = set()
    for e in R.served_models().values():
        a = e["arch"]
        tower = next((t for t in a.values() if isinstance(t, dict) and "image_size" in t), None)
        if tower is not None and (a.get("resize_mode") or "crop") == mode:
            sizes.add(tower["image_size"])
    return sorted(sizes)


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
