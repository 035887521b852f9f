"""The GEMM at the shapes and edges where its two kernels go wrong, each case pinned to the kernel it runs.

The library runs the persistent 128 x 256 kernel for K >= 1024, N % 256 == 0 and at least one 128 x 256 tile per SM,
and the 128 x 128 kernel otherwise (gemm.cu launch()).  b200_debug_gemm reports which one ran and takes the SM
count the rule is applied with, so a small count sends small shapes to the persistent kernel with each CTA walking
many tiles, and a huge one sends any shape to the 128 x 128 kernel: no case runs a kernel where the rule would not.

Every case writes into a larger buffer whose rows >= M and columns >= N hold a sentinel that must survive.  The
reference is torch fp64 on the bf16-rounded operands, on the GPU so that the served shapes stay fast."""
import itertools
import math

import pytest
import torch

from _checks import bf16
from marqo_b200 import model_registry
from marqo_b200._native import GEMM_128x128, GEMM_PERSISTENT

pytestmark = pytest.mark.gpu

SENTINEL = -7.5      # exact in bf16 and fp32
GUARD_ROWS, GUARD_COLS = 5, 40
ALL_128x128 = 100_000            # an SM count no shape reaches a full wave of: the 128 x 128 kernel
KERNEL_NAME = {GEMM_128x128: "128x128", GEMM_PERSISTENT: "persistent"}
NONE, GELU, QUICKGELU = 0, 1, 2
ACT_NAME = {NONE: "", GELU: "-gelu", QUICKGELU: "-quickgelu"}


@pytest.fixture(scope="module")
def sm_count(gpu_required):
    n = torch.cuda.get_device_properties(0).multi_processor_count
    assert n > 16, "the served-shape cases assume one 16-token query cannot fill a wave"
    return n


def _act(z: torch.Tensor, act: int) -> torch.Tensor:
    if act == GELU:
        return 0.5 * z * (1.0 + torch.erf(z / math.sqrt(2.0)))
    if act == QUICKGELU:
        return z * torch.sigmoid(1.702 * z)
    return z


def _run(M, N, K, act, out_bf16, residual, sms, seed, bias=True, alt_sms=None):
    """One GEMM into a guarded buffer, checked against fp64 -> (buffer, kernel), and (buffer, kernel) of a second run
    of the same inputs with SM count alt_sms when given."""
    from marqo_b200.engine import debug_gemm_into
    g = torch.Generator().manual_seed(seed)
    A = bf16(torch.randn(M, K, generator=g))
    W = bf16(torch.randn(N, K, generator=g) / math.sqrt(K))
    b = torch.randn(N, generator=g) if bias else None
    io = torch.full((M + GUARD_ROWS, N + GUARD_COLS), SENTINEL)
    res = torch.randn(M, N, generator=g)
    if residual:
        io[:M, :N] = res
    args = (A.numpy(), W.numpy(), io.numpy(), None if b is None else b.numpy())
    kw = dict(act=act, out_bf16=bool(out_bf16), residual_in_place=residual, return_kernel=True)
    got, kernel = debug_gemm_into(*args, sms=sms, **kw)
    got = torch.from_numpy(got)
    z = A.cuda().double() @ W.cuda().double().t()
    if b is not None:
        z = z + b.cuda().double()
    ref = _act(z, act)
    if residual:
        ref = ref + res.cuda().double()
    if out_bf16:
        torch.testing.assert_close(got[:M, :N].cuda().double(), ref, rtol=1e-2, atol=1e-2)   # bf16 output rounding
    else:
        torch.testing.assert_close(got[:M, :N].cuda().double(), ref, rtol=2e-4, atol=3e-4)
    assert bool((got[M:, :] == SENTINEL).all()), "rows >= M were written"
    assert bool((got[:, N:] == SENTINEL).all()), "columns >= N were written"
    if alt_sms is None:
        return (got, kernel), None
    alt, alt_kernel = debug_gemm_into(*args, sms=alt_sms, **kw)
    return (got, kernel), (torch.from_numpy(alt), alt_kernel)


def _check_same_bits(got, alt):
    """The 128 x 128 and the persistent kernel sum each output in the same k order and share the epilogue: the whole
    buffer, guards included, must be bitwise the same."""
    assert alt[1] == GEMM_128x128, f"SM count {ALL_128x128} ran the {KERNEL_NAME.get(alt[1], alt[1])} kernel"
    same = got[0].view(torch.int32) == alt[0].view(torch.int32)
    if not bool(same.all()):
        r, c = (~same).nonzero()[0].tolist()
        pytest.fail(f"{int((~same).sum())} elements differ between the kernels, first at ({r}, {c}): persistent "
                    f"{float(got[0][r, c])!r}, 128x128 {float(alt[0][r, c])!r}")


def _assert_kernel(kernel, expected):
    assert kernel == expected, f"ran the {KERNEL_NAME.get(kernel, kernel)} kernel, expected {KERNEL_NAME[expected]}"


# --------------------------------------------------------------------------------------------- (a) the selection rule
@pytest.mark.parametrize("M,N,K,expected", [
    (128, 1024, 1024, GEMM_PERSISTENT),   # 4 tiles of 128 x 256 = 4 SMs: one full wave
    (128, 768, 1024, GEMM_128x128),       # 3 tiles: less than a wave
    (128, 1024, 960, GEMM_128x128),       # K < 1024
    (128, 640, 1024, GEMM_128x128),       # N % 256 != 0
], ids=["persistent-4tiles", "128x128-3tiles", "128x128-K960", "128x128-N640"])
def test_selection_rule_with_4_sms(gpu_required, M, N, K, expected):
    (_, kernel), _ = _run(M, N, K, NONE, 0, True, 4, seed=M + N + K)
    _assert_kernel(kernel, expected)


@pytest.mark.parametrize("extra_rows,expected", [(0, GEMM_128x128), (1, GEMM_PERSISTENT)],
                         ids=["128x128-one-tile-short", "persistent-exactly-one-wave"])
def test_selection_rule_on_the_device(sm_count, extra_rows, expected):
    """N = 256: one tile per 128 rows.  sms=None applies the rule with the device's own SM count."""
    M = 128 * (sm_count - 1) + extra_rows
    (_, kernel), _ = _run(M, 256, 1024, NONE, 0, True, None, seed=M)
    _assert_kernel(kernel, expected)


# ------------------------------------------------------------------------------------- (b) persistent tile walks
# Epilogue instantiations (act, out_bf16, residual in place); the fp32 residual stream updated in place comes twice.
EPILOGUES = [(NONE, 0, True), (GELU, 1, False), (NONE, 1, False), (QUICKGELU, 0, False), (NONE, 0, True),
             (QUICKGELU, 1, False), (GELU, 0, True)]
TAIL_ROWS = [1, 64, 65, 127]   # M % 128: the last row tile holds 1, 64, 65 or 127 rows


def _walk_cases():
    """sms x N x K, with the last row tile's height and the epilogue cycling through their lists.  K = 1024, 1088,
    1152, 1344, 3072: 16, 17, 18, 21 and 48 k-blocks, every residue mod the 3-stage ring, so a tile starts on each
    stage and with each mbarrier phase.  The tile count is at least 2 sms + 1, so every CTA walks two or more tiles,
    and not a multiple of sms where the column tiles allow it, so that some CTAs walk one more than others."""
    cases = []
    for i, (sms, N, K) in enumerate(itertools.product([1, 2, 5], [256, 768, 1024], [1024, 1088, 1152, 1344, 3072])):
        tiles_n = N // 256
        tiles_m = -(-(2 * sms + 1) // tiles_n)
        while tiles_n % sms != 0 and (tiles_m * tiles_n) % sms == 0:
            tiles_m += 1
        M = 128 * (tiles_m - 1) + TAIL_ROWS[i % len(TAIL_ROWS)]
        act, out_bf16, residual = EPILOGUES[i % len(EPILOGUES)]
        ep = ("bf16" if out_bf16 else "fp32") + ACT_NAME[act] + ("-res" if residual else "")
        cases.append(pytest.param(sms, M, N, K, act, out_bf16, residual,
                                  id=f"persistent-sms{sms}-M{M}-N{N}-K{K}-{ep}"))
    return cases


@pytest.mark.parametrize("sms,M,N,K,act,out_bf16,residual", _walk_cases())
def test_persistent_tile_walk(gpu_required, sms, M, N, K, act, out_bf16, residual):
    got, alt = _run(M, N, K, act, out_bf16, residual, sms, seed=sms * 100003 + M * 7 + N + K, alt_sms=ALL_128x128)
    _assert_kernel(got[1], GEMM_PERSISTENT)
    _check_same_bits(got, alt)


# ----------------------------------------------------------------------------------------- (c) served layer shapes
def _served_layers():
    """{(width, mlp): {act}} of every encoder tower in the model registry (CLIP vision and text, the BERTs, MPNet)."""
    layers = {}
    for entry in model_registry.all_models().values():
        arch = entry["arch"]
        if "vision" in arch:
            act = QUICKGELU if arch["act"] == "quickgelu" else GELU
            towers = [arch["vision"], arch["text"]]
        else:
            act, towers = GELU, [arch]
        for t in towers:
            layers.setdefault((t["width"], t["mlp"]), set()).add(act)
    return layers


def _served_cases():
    """The four layer GEMMs of every served width at M = 16 (one 16-token query) and 77 (CLIP text), and, for those
    the persistent kernel can take, at M one row tile short of a full wave of 128 x 256 tiles on the device
    ("below"), at the fewest rows that fill the wave ("wave") and at a wave and a half with a partial last row tile
    ("wave+")."""
    cases = []
    for (w, mlp), acts in sorted(_served_layers().items()):
        gemms = [("qkv", 3 * w, w, NONE, 1, False), ("out_proj", w, w, NONE, 0, True)]
        gemms += [("fc1" + ACT_NAME[a], mlp, w, a, 1, False) for a in sorted(acts)]
        gemms += [("fc2", w, mlp, NONE, 0, True)]
        for name, N, K, act, out_bf16, residual in gemms:
            ms = ["16", "77"]
            if K >= 1024 and N % 256 == 0:
                ms += ["below", "wave", "wave+"]
            for m in ms:
                kernel = GEMM_PERSISTENT if m in ("wave", "wave+") else GEMM_128x128
                cases.append(pytest.param(w, m, N, K, act, out_bf16, residual, kernel,
                                          id=f"{KERNEL_NAME[kernel]}-w{w}-{name}-M{m}"))
    return cases


def test_served_cases_cover_fc2_at_768():
    """fc2 of the 768-wide models (three 256-wide column tiles) is among the persistent served cases."""
    ids = [c.id for c in _served_cases()]
    assert {w for (w, _) in _served_layers()} == {384, 512, 768, 1024}
    assert "persistent-w768-fc2-Mwave" in ids and "persistent-w768-fc2-Mwave+" in ids


@pytest.mark.parametrize("w,m,N,K,act,out_bf16,residual,expected", _served_cases())
def test_served_layer_shape(sm_count, w, m, N, K, act, out_bf16, residual, expected):
    rows_per_wave = -(-sm_count // (N // 256)) if N % 256 == 0 else None
    M = {"16": 16, "77": 77}.get(m)
    if M is None:
        wave = 128 * rows_per_wave
        M = {"below": wave - 128, "wave": wave, "wave+": wave + wave // 2 + 37}[m]
    persistent = expected == GEMM_PERSISTENT
    got, alt = _run(M, N, K, act, out_bf16, residual, None, seed=M * 7 + N + K + act,
                    alt_sms=ALL_128x128 if persistent else None)
    _assert_kernel(got[1], expected)
    if persistent:
        _check_same_bits(got, alt)


# ------------------------------------------------------------------------------------------- (d) 128 x 128 edges
@pytest.mark.parametrize("residual", [True, False], ids=["fp32-res", "bf16"])
@pytest.mark.parametrize("N", [32, 160])
@pytest.mark.parametrize("M", [1, 8, 16, 63, 65])
def test_128x128_edges(gpu_required, M, N, residual):
    """A single 32-column tile, and a full tile plus a 32-column one (for a bf16 output a partial 64-column box), at
    latency-sized M; with the fp32 residual in place, or a bf16 output with an activation."""
    act = NONE if residual else (GELU, QUICKGELU)[M % 2]
    (_, kernel), _ = _run(M, N, 256, act, 0 if residual else 1, residual, None, seed=M * 1000 + N + residual)
    _assert_kernel(kernel, GEMM_128x128)


# ------------------------------------------------------------------------------------ (f) activations at the edges
EDGE_VALUES = [0.0, 1e-7, 1e-5, 1e-3, 1.0, 3.0, 10.0, 400.0, 65000.0, 65530.0, 7e4, 1e5]
QUICKGELU_TAIL = [-60.0, -100.0, -1000.0]   # 2^(1.702 log2(e) |z|) overflows fp32


def _edge_bias(n: int) -> torch.Tensor:
    """The edge values with both signs, then a dense sweep of [-12, 12] in the remaining columns."""
    vals = [s * v for v in EDGE_VALUES for s in (1.0, -1.0)] + QUICKGELU_TAIL
    return torch.cat([torch.tensor(vals), torch.linspace(-12.0, 12.0, n - len(vals))]).float()


def _edge_bound(z: torch.Tensor, ref: torch.Tensor, act: int, out_bf16: int) -> torch.Tensor:
    """The error each epilogue is documented to keep (gemm.cu), per element."""
    if act == GELU and out_bf16:
        # gelu_erf_h2: bf16 rounding, the fp16 evaluation (roundings of 2^-11 scaled by |z| / 2), the fp16 subnormal
        # spacing
        return 2.0 ** -8 * ref.abs() + 2.0 ** -9 * z.abs() + 2.0 ** -24
    if act == GELU:
        # gelu_erf: erf to 1.9e-5 absolute (scaled by |z| / 2), ex2.approx's 2^-22 on top, then fp32 rounding
        return (1.9e-5 + 2.0 ** -22) * z.abs() / 2 + 2.0 ** -22 * ref.abs()
    # quick_gelu: ex2.approx's 2^-22 and the fp32 rounding of its argument 1.702 log2(e) z (2^-23 relative, so
    # 2^-23 |argument| absolute in the exponent); the quotient flushes to zero below 2^-126 (ftz)
    bound = (2.0 ** -21 + 2.0 ** -22 * (1.702 * math.log2(math.e)) * z.abs()) * ref.abs() + 2.0 ** -126 * (1 + z.abs())
    return bound + 2.0 ** -8 * ref.abs() if out_bf16 else bound


@pytest.mark.parametrize("sms,expected", [(4, GEMM_PERSISTENT), (ALL_128x128, GEMM_128x128)],
                         ids=["persistent", "128x128"])
@pytest.mark.parametrize("act,out_bf16", [(GELU, 1), (GELU, 0), (QUICKGELU, 1), (QUICKGELU, 0)],
                         ids=["bf16-gelu", "fp32-gelu", "bf16-quickgelu", "fp32-quickgelu"])
def test_activation_edges(gpu_required, act, out_bf16, sms, expected):
    """A = 0 so that z = bias exactly; every output finite and within the bound of its epilogue."""
    from marqo_b200.engine import debug_gemm_into
    M, N, K = 128, 1024, 1024
    z = _edge_bias(N)
    io = torch.full((M + GUARD_ROWS, N + GUARD_COLS), SENTINEL)
    got, kernel = debug_gemm_into(torch.zeros(M, K).numpy(), torch.ones(N, K).numpy(), io.numpy(), z.numpy(), act=act,
                                  out_bf16=bool(out_bf16), sms=sms, return_kernel=True)
    _assert_kernel(kernel, expected)
    got = torch.from_numpy(got)
    assert bool((got[M:, :] == SENTINEL).all()) and bool((got[:, N:] == SENTINEL).all()), "the guards were written"
    got = got[:M, :N].double()
    y, zd = got[0], z.double()
    bad = ~torch.isfinite(got).all(0)
    assert not bool(bad.any()), f"non-finite outputs: z = {zd[bad].tolist()} -> {y[bad].tolist()}"
    assert bool((got == y).all()), "rows with the same z differ"
    ref = _act(zd, act)
    err, bound = (y - ref).abs(), _edge_bound(zd, ref, act, out_bf16)
    over = err > bound
    assert not bool(over.any()), (f"outside the bound: z = {zd[over].tolist()[:8]} -> {y[over].tolist()[:8]}, "
                                  f"reference {ref[over].tolist()[:8]}; worst error / bound {float((err / bound).max())}")
