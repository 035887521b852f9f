"""The scan's error bound eps (score.cu, query_prep_kernel) checked against the tensor core's real error.

Every search is exact because of one number: eps[q] bounds |approximate scan key - exact scan key| for every row,
and the merge guard and the collect threshold both rest on it.  b200_debug_index_last_scan hands back what the last
search left on the device: eps, the fp16 query block as scanned, and every scan CTA's list of its 16 best
(approximate key, row) per query.

The corpora here have at most `grid` 128-row tiles with exactly 16 live rows each, every row its own document, so
each CTA scans one tile and lists all of its live rows for every query: every (query, live row) approximate key is
observed and compared with the exact scan-domain key computed in fp64 from the stored rows.  The input families are
built to come near the bound; each asserts a floor on its worst ratio |approx - exact| / eps, half the worst ratio
measured on an NVIDIA H100 80GB HBM3 (700 W power limit), so a family that stops reaching the bound fails.

The staircase family pins the accumulation model.  The first 16 coordinates are 32, so the first k-step of a
self-match leaves the fp32 accumulator at exactly 2^14 (ulp 2^-9); every other coordinate is T, the largest fp16 with
T^2 < 2^-9.  Truncating each addend against the accumulator would lose every tail product, (d - 16) 2^-9 against
eps ~ d 2^-8, a ratio near 0.5.  The H100 loses a quarter of that, ratio 0.124 at d = 4096: each group of four
products is added exactly and the sum truncated once (4 T^2 is just under 4 ulp, so each group drops almost one ulp).
With the tail of the query negated the sum falls below 2^14, into the binade whose ulp is 2^-10, and the loss halves
(0.062): the truncation rounds toward zero.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TILE = 128          # rows per scan tile
LIVE = 16           # live rows per tile = entries per (CTA, query) list
TILES = 16          # tiles per corpus (fewer than the H100's SMs: one tile per scan CTA)
NQ = 32
METRICS = ["prenormalized-angular", "angular", "dotproduct", "euclidean"]
DIMS = [64, 768, 1024, 1088, 4096]   # 1024: the widest resident query block; above it the streamed kernel
T = np.float32(1448 * 2.0 ** -15)    # largest fp16 with T^2 < 2^-9
assert float(T) ** 2 < 2.0 ** -9 and float(np.nextafter(np.float16(T), np.float16(1))) ** 2 >= 2.0 ** -9
NORMALISED = ("prenormalized-angular", "angular")

# Floors of the adversarial families: half the smallest worst ratio measured on an H100 over the family's dims (the
# range of worst ratios from d = 64 to 4096 follows each entry).
FLOORS = {
    ("staircase", "prenormalized-angular"): 0.046,       # 0.0935 .. 0.124
    ("staircase", "angular"): 0.046,                     # 0.0935 .. 0.124
    ("staircase", "dotproduct"): 0.046,                  # 0.0935 .. 0.124
    ("staircase", "euclidean"): 0.036,                   # 0.0721 .. 0.0993
    ("staircase_negated", "prenormalized-angular"): 0.031,   # 0.0622 .. 0.0623
    ("staircase_negated", "angular"): 0.031,             # 0.0622 .. 0.0623
    ("staircase_negated", "dotproduct"): 0.031,          # 0.0622 .. 0.0623
    ("staircase_negated", "euclidean"): 0.024,           # 0.048 .. 0.0497
    ("cancellation", "prenormalized-angular"): 0.0072,   # 0.0145 .. 0.0211
    ("cancellation", "angular"): 0.0076,                 # 0.0153 .. 0.0207
    ("cancellation", "dotproduct"): 0.0071,              # 0.0143 .. 0.0214
    ("cancellation", "euclidean"): 0.0054,               # 0.0108 .. 0.0168
    ("fp16_extremes", "dotproduct"): 0.00012,            # 0.00672 at d = 64 .. 0.000244 at 4096
    ("fp16_extremes", "euclidean"): 0.000069,            # 0.00632 at d = 64 .. 0.00014 at 4096
    ("euclidean_large", "euclidean"): 0.0065,            # 0.0131 .. 0.0162
    ("modifiers", "prenormalized-angular"): 0.0082,      # 0.0166 .. 0.0186
    ("modifiers", "angular"): 0.0014,                    # 0.00281 at d = 64 .. 0.0908 at 4096
    ("modifiers", "dotproduct"): 0.0094,                 # 0.019 .. 0.0224
    ("modifiers", "euclidean"): 0.018,                   # 0.0373 .. 0.113
}


def _f16(x):
    return np.asarray(x, np.float32).astype(np.float16).astype(np.float32)


def _closeness(dot, metric):
    """closeness_from_dot in fp64: `dot` is the dot product, or minus the squared distance (euclidean)."""
    if metric == "euclidean":
        return 1.0 / (1.0 + np.sqrt(np.maximum(-dot, 0.0)))
    if metric == "prenormalized-angular":
        return 1.0 / (1.0 + (1.0 - dot))
    if metric == "angular":
        return 1.0 / (1.0 + np.arccos(np.clip(dot, -1.0, 1.0)))
    return dot


# ------------------------------------------------------------------------------------------------ input families
# Each returns (live rows fp32 [TILES * LIVE, d], queries fp32 [NQ, d], per-row (mult, add) or None).
def _gaussian(rng, metric, d):
    rows = rng.standard_normal((TILES * LIVE, d)).astype(np.float32)
    rows /= np.linalg.norm(rows, axis=1, keepdims=True)
    if metric not in NORMALISED:
        rows *= np.float32(3.0)
    q = rng.standard_normal((NQ, d)).astype(np.float32)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    q[: NQ // 2] = rows[rng.choice(len(rows), NQ // 2, replace=False)]
    return rows, q, None


def _staircase(rng, metric, d, negate_tail=False):
    sign = np.where(rng.random((TILES * LIVE, d)) < 0.5, -1.0, 1.0).astype(np.float32)
    rows = np.full((TILES * LIVE, d), T, np.float32)
    rows[:, :16] = 32.0
    rows *= sign
    if metric in NORMALISED:
        rows *= np.float32(2.0 ** -7)   # 16 * 0.25^2 = 1: a unit self-match
    q = rows[rng.choice(len(rows), NQ, replace=False)].copy()   # q = e
    if negate_tail:   # truncation of a negative addend rounds toward zero
        q[:, 16:] *= -1
    return rows, q, None


def _staircase_negated(rng, metric, d):
    return _staircase(rng, metric, d, negate_tail=True)


def _cancellation(rng, metric, d):
    """e = [x, -x] and q = [x', x']: the accumulator climbs to |x|^2 over the first half and cancels over the second."""
    h = d // 2
    x = _f16(rng.standard_normal((TILES * LIVE, h)) * (1.0 / np.sqrt(d) if metric in NORMALISED else 4.0))
    rows = np.concatenate([x, -x], axis=1)
    pick = rng.choice(len(rows), NQ, replace=False)
    q = np.concatenate([x[pick], x[pick]], axis=1)
    q[NQ // 2:, h:] *= -1   # half the queries are self-matches: every product positive
    return rows, q, None


def _fp16_extremes(rng, metric, d):
    """+-65504 beside fp16 subnormals (dot product and euclidean only: the normalised metrics take unit rows)."""
    n = TILES * LIVE
    sub = rng.integers(1, 1024, size=(n, d)).astype(np.float32) * np.float32(2.0 ** -24)
    big = rng.random((n, d)) < 0.125
    rows = np.where(big, np.float32(65504.0), sub)
    rows *= np.where(rng.random((n, d)) < 0.5, -1.0, 1.0).astype(np.float32)
    q = rows[rng.choice(n, NQ, replace=False)].copy()
    flip = rng.random((NQ // 2, d)) < 0.5
    q[: NQ // 2] = np.where(flip & (np.abs(q[: NQ // 2]) < 1.0), -q[: NQ // 2], q[: NQ // 2])
    return rows, q, None


def _euclidean_large(rng, metric, d):
    """Rows of norm ~40 sqrt(d) and q ~ e / 2: 2 q.e ~ |e|^2, so the key is a small difference of large fp32 terms."""
    rows = _f16(rng.standard_normal((TILES * LIVE, d)) * 40.0)
    q = rows[rng.choice(len(rows), NQ, replace=False)] * np.float32(0.5)
    q += rng.standard_normal(q.shape).astype(np.float32) * np.float32(0.01)
    return rows, q, None


def _modifiers(rng, metric, d):
    """mult up to 1e3, add up to 1e4, near self-matches: acos is steep near 1, and prenormalised rows and queries of
    norm 1.39 leave 2 - qn R close to the 0.05 room the bound requires."""
    n = TILES * LIVE
    rows = rng.standard_normal((n, d)).astype(np.float32)
    rows /= np.linalg.norm(rows, axis=1, keepdims=True)
    q = rows[rng.choice(n, NQ, replace=False)] + rng.standard_normal((NQ, d)).astype(np.float32) * np.float32(
        1e-3 / np.sqrt(d))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    if metric == "prenormalized-angular":
        rows *= np.float32(1.39)
        q *= np.float32(1.39)
    elif metric != "angular":
        rows *= np.float32(2.0)
        q *= np.float32(2.0)
    mult = rng.uniform(1.0, 1e3, n)
    add = rng.uniform(-1e4, 1e4, n)
    return rows, q, (mult, add)


FAMILIES = {
    "gaussian": (_gaussian, METRICS),
    "staircase": (_staircase, METRICS),
    "staircase_negated": (_staircase_negated, METRICS),
    "cancellation": (_cancellation, METRICS),
    "fp16_extremes": (_fp16_extremes, ["dotproduct", "euclidean"]),
    "euclidean_large": (_euclidean_large, ["euclidean"]),
    "modifiers": (_modifiers, METRICS),
}
CASES = [(f, m, d, False) for f, (_, ms) in FAMILIES.items() for m in ms for d in DIMS]
CASES += [(f, m, 768, True) for f, (_, ms) in FAMILIES.items() for m in ms]


def _scan_keys(store, metric, pos, mods):
    """-> (approx [nq, L], exact [nq, L], eps [nq]) over the L live rows `pos` (sorted) of the last search."""
    from marqo_b200.engine import debug_last_scan
    s = debug_last_scan(store)
    tiles = len(pos) // LIVE
    assert s["grid"] == tiles, s["grid"]
    # every CTA listed exactly the live rows of its tile, for every query
    listed = np.sort(s["list_row"], axis=2)
    np.testing.assert_array_equal(listed, np.broadcast_to(pos.reshape(tiles, 1, LIVE), listed.shape))
    np.testing.assert_array_equal(s["list_doc"], s["list_row"])
    nq = s["nq"]
    idx = np.searchsorted(pos, s["list_row"])                       # [grid, nq, LIVE] -> live row index
    approx = np.empty((nq, len(pos)))
    approx[np.arange(nq)[None, :, None], idx] = s["list_score"].astype(np.float64)
    e = store.get_rows(pos).astype(np.float64)
    qv = s["queries"].astype(np.float64)
    dot = qv @ e.T
    n2e = (e * e).sum(axis=1)
    if metric == "euclidean":
        key = 2.0 * dot - n2e[None, :]
        dot = -((qv * qv).sum(axis=1)[:, None] - key)               # minus the squared distance
    else:
        key = dot
    if mods is not None:
        mult, add = mods
        key = mult[pos][None, :] * _closeness(dot, metric) + add[pos][None, :]
    return approx, key, s["eps"].astype(np.float64)


def _worst_ratio(family, metric, d, streamed, seed=0):
    from marqo_b200 import _native as N
    from marqo_b200.engine import RowStore, debug_scan_kernel
    rng = np.random.default_rng([seed, d, METRICS.index(metric), list(FAMILIES).index(family)])
    rows, q, mods = FAMILIES[family][0](rng, metric, d)
    n = TILES * TILE
    pos = np.sort(np.stack([t * TILE + rng.choice(TILE, LIVE, replace=False) for t in range(TILES)]), axis=1).ravel()
    corpus = np.zeros((n, d), np.float32)           # dead rows are zero: they do not raise the stored maximum norm
    corpus[pos] = rows
    store = RowStore(d, metric=metric)
    try:
        if streamed:
            debug_scan_kernel(store, force_streamed=True)
        store.add(corpus, np.arange(n, dtype=np.int32))
        store.delete_rows(np.setdiff1d(np.arange(n), pos))
        full = None
        kw = {}
        if mods is not None:
            full = tuple(np.zeros(n) for _ in range(2))
            full[0][pos], full[1][pos] = mods
            store.set_attributes(0, pos, full[0][pos])
            store.set_attributes(1, pos, full[1][pos])
            kw = dict(mult=[(0, 1.0)], add=[(1, 1.0)])
        store.search(q, 10, **kw)
        want = N.SCAN_STREAMED_Q if streamed or d > 1024 else N.SCAN_RESIDENT_Q
        assert debug_scan_kernel(store) == want
        approx, exact, eps = _scan_keys(store, metric, pos, full)
    finally:
        store.close()
    err = np.abs(approx - exact)
    bad = err > eps[:, None]
    assert not bad.any(), (
        f"{family} {metric} d={d}: |approx - exact| exceeds eps for {int(bad.sum())} pairs; worst ratio "
        f"{float((err / eps[:, None]).max()):.4g}")
    return float((err / eps[:, None]).max())


@pytest.mark.parametrize("family,metric,d,streamed", CASES,
                         ids=[f"{f}-{m}-{d}{'-streamed' if s else ''}" for f, m, d, s in CASES])
def test_scan_error_within_eps(gpu_required, family, metric, d, streamed):
    ratio = _worst_ratio(family, metric, d, streamed)
    floor = FLOORS.get((family, metric))
    if floor is not None:
        assert ratio >= floor, f"{family} {metric} d={d}: worst ratio {ratio:.4g} no longer reaches {floor}"


# ------------------------------------------------------------------------------------------------ end to end
def _head_row(d, bumps):
    """Head coordinates 32 with +2^-5 / -2^-6 steps (q.e moves by +1 / -0.5 against a staircase head), tail zero: the
    tensor core sums such rows exactly."""
    r = np.zeros(d, np.float32)
    r[:16] = 32.0
    for i, b in enumerate(bumps):
        r[i] += b
    return r


@pytest.mark.parametrize("streamed", [False, True], ids=["resident", "streamed"])
def test_inverted_approximate_order_is_settled_exactly(gpu_required, score_oracle, streamed):
    """A staircase self-match S (exact q.e = 2^14 + 1008 T^2 ~ 2^14 + 1.968) against a row C of exact key 2^14 + 1.5
    that the tensor core sums exactly.  The scan loses ~0.49 of S (the staircase ratio 0.123 at d = 1024, measured
    above), more than the 0.47 gap, so its approximate order is inverted; the guard must flag the query and the exact
    pass return S first.  Forty more rows of keys 2^14 - 0.5 .. 2^14 + 1.5 fill two tiles' lists."""
    from marqo_b200 import _native as N
    from marqo_b200.engine import RowStore, debug_last_scan, debug_scan_kernel
    d, tiles = 1024, 20
    rng = np.random.default_rng(5)
    n = tiles * TILE
    corpus = rng.standard_normal((n, d)).astype(np.float32)
    s_row, c_row = 5, 77
    corpus[s_row] = T
    corpus[s_row, :16] = 32.0
    c_bumps = [2.0 ** -5, 2.0 ** -5, -2.0 ** -6]                      # +1 +1 -0.5
    corpus[c_row] = _head_row(d, c_bumps)
    steps = [[], [-2.0 ** -6], [2.0 ** -5], c_bumps]                  # keys 2^14 + {0, -0.5, 1, 1.5}
    competitors = rng.choice(np.arange(TILE, 3 * TILE), 40, replace=False)
    for r in competitors:
        corpus[r] = _head_row(d, steps[rng.integers(len(steps))])
    q = rng.standard_normal((3, d)).astype(np.float32)
    q[0] = corpus[s_row]
    store = RowStore(d, metric="dotproduct")
    try:
        store.add(corpus)
        if streamed:
            debug_scan_kernel(store, force_streamed=True)
        e = store.get_rows([s_row, c_row]).astype(np.float64)
        exact = e @ e[0]
        assert exact[1] == 2.0 ** 14 + 1.5 and exact[0] > exact[1], exact
        for k in (1, 10):
            flagged = store.search_stats()["flagged"]
            got = store.search(q, k)
            assert debug_scan_kernel(store) == (N.SCAN_STREAMED_Q if streamed else N.SCAN_RESIDENT_Q)
            s = debug_last_scan(store)
            lst = s["list_row"][0, 0], s["list_score"][0, 0]               # CTA 0 scanned tile 0 alone
            approx = {r: float(lst[1][list(lst[0]).index(r)]) for r in (s_row, c_row)}
            assert approx[c_row] == exact[1] and approx[s_row] < approx[c_row], approx
            assert store.search_stats()["flagged"] > flagged
            edoc, erow, escore = score_oracle.search(q, corpus, k, "dotproduct")
            np.testing.assert_array_equal(got[0], edoc)
            np.testing.assert_array_equal(got[1], erow)
            np.testing.assert_array_equal(got[2], escore)
            assert got[0][0, 0] == s_row
    finally:
        store.close()


# ------------------------------------------------------------------------------------------------ max_n2
def _eps_floor(metric, d, qv, max_n2):
    """query_prep_kernel's eps in float32 for the fp16 query qv, with R from the largest squared norm `max_n2` of the
    live stored rows.  The device multiplies sqrt(max_n2) by 1.001 to cover the rounding of its fp32 norm sums; that
    margin is left out here, so the device's eps is at least this whenever its max_n2 covers every live row."""
    f = np.float32
    qn = f(np.sqrt(f(np.sum(qv.astype(np.float64) ** 2)))) * f(1.001)
    R = f(np.sqrt(f(max_n2)))
    c = f(d) * f(2.0 ** -22)
    eps = c * qn * R
    if metric == "euclidean":
        eps = f(2) * eps + f(0.5) * c * R * R + f(2.0 ** -21) * (f(2) * qn * R + R * R)
    return eps


@pytest.mark.parametrize("metric", ["dotproduct", "euclidean"])
def test_eps_covers_the_largest_live_row(gpu_required, metric, tmp_path):
    """eps reads max_n2, the largest stored squared norm.  After every way rows reach the store, eps must be at least
    the bound for the largest norm among the live rows (a stale, larger max_n2 is allowed).  Each step adds a row
    twice as long as any before, so an update that is missed leaves eps too small."""
    import torch
    from marqo_b200 import _native as N
    from marqo_b200.engine import RowStore, debug_last_scan
    d = 256
    rng = np.random.default_rng(9)
    probe = rng.standard_normal((1, d)).astype(np.float32)
    scale = [1.0]

    def batch(m, grow=True):
        x = rng.standard_normal((m, d)).astype(np.float32)
        x /= np.linalg.norm(x, axis=1, keepdims=True)
        x *= np.float32(scale[0])
        if grow:
            scale[0] *= 2.0
            x[rng.integers(m)] *= np.float32(2.0)   # one row longer than the rest
        return x

    def check(st, step):
        st.search(probe, 1)
        s = debug_last_scan(st)
        live = np.flatnonzero(alive[: len(st)])
        rows = st.get_rows(live).astype(np.float64)
        want = _eps_floor(metric, d, s["queries"][0], (rows * rows).sum(axis=1).max())
        assert s["eps"][0] >= want, f"after {step}: eps {s['eps'][0]} < {want}"

    store = RowStore(d, metric=metric, capacity=512)
    alive = np.zeros(1 << 12, bool)
    try:
        store.add(batch(200), np.arange(200, dtype=np.int32))
        alive[:200] = True
        check(store, "add")
        x = torch.from_numpy(batch(100)).cuda()
        ids = torch.arange(200, 300, dtype=torch.int32, device="cuda")
        store.add_device(x.data_ptr(), 100, ids.data_ptr())
        alive[200:300] = True
        check(store, "add_device")
        x = torch.from_numpy(batch(100)).cuda()
        store.add_device_docs(x.data_ptr(), np.arange(300, 400, dtype=np.int32))
        torch.cuda.synchronize()
        alive[300:400] = True
        check(store, "add_device_docs")
        store.add(batch(300), np.arange(400, 700, dtype=np.int32))   # past the 512-row capacity
        alive[400:700] = True
        check(store, "growth past capacity")
        path = str(tmp_path / "n2.b200idx")
        store.save(path)
        back = RowStore.load(path)
        try:
            check(back, "save / load")
        finally:
            back.close()
        dead = rng.choice(700, 150, replace=False)
        store.delete_rows(dead)
        alive[dead] = False
        new_of_old = store.compact()
        alive[:] = False
        alive[: int((new_of_old >= 0).sum())] = True
        check(store, "compact")
        n2 = (store.get_rows(np.arange(len(store))).astype(np.float64) ** 2).sum(axis=1)
        top = int(np.argmax(n2))
        store.delete_rows([top])
        alive[top] = False
        check(store, "deleting the largest row")
        n = len(store)
        bad = batch(2)
        bad[1, 0] = np.nan
        with pytest.raises(N.NativeError) as e:
            store.add(bad, np.array([n, n + 1], np.int32))
        assert e.value.code == N.ERR_INVALID_ARG and len(store) == n
        check(store, "a rejected batch")
        # a reloaded store sees only what was saved: its eps must still cover its own largest row
        store.save(path)
        back = RowStore.load(path)
        try:
            check(back, "a reload after compaction")
        finally:
            back.close()
    finally:
        store.close()
