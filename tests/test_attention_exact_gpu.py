"""Attention checked exactly where it can be, and against an fp64 error bound everywhere else.

Both kernels (attention.cuh: mma.sync for S < 128, wgmma for S >= 128) share four properties that make most of their
behaviour checkable bit for bit:

- a masked score is replaced by -inf with a select, so its p is exp2f(-inf) = 0 and its bf16 P is exactly 0, whatever
  the key held;
- 0 * v = 0 for finite v, and adding exact zeros leaves an exact sum unchanged, so the tensor core rounds every group
  of products the same way;
- in a block where all of a row's keys are masked the row maximum does not move, so corr = exp2f(0) = 1 and row_sum
  and o are unchanged;
- each output row depends only on its own query row: the CTA of query i is blockIdx.x = i / 64 whatever S is, and the
  key blocks start at key 0.

So, with the same kernel on both sides, a key-length mask equals keys overwritten with huge finite values, equals the
sequence cut at that length, equals the causal mask row by row; a sequence is unaffected by its neighbours in the
batch; heads are independent; and a row without keys is +0.  The tests below assert those with bitwise equality,
at the key lengths and rows where the 64- and 128-key tiles end.  b200_debug_attention runs on device buffers the
test owns, so the output can sit between guard rows and start out as NaN: every element must be written, and nothing
outside it.

Where results are not exact, each output element is held to a bound derived from the kernel's arithmetic (see
_bound), at every attention shape the model registry serves (the key-length towers, whose S is the batch's longest
text, at the tile edges of both kernels and at their token limits), on input families built to come near it.  Each
adversarial family asserts a floor on its worst ratio error / bound, half the worst ratio measured on an NVIDIA H100
80GB HBM3 (700 W power limit), so a bound that stops being tight is noticed.  map_attention (the SigLIP MAP head and
the ResNet attention pool) gets the same bound without the rounding of P, which it keeps in fp32.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from marqo_b200 import _native as N
from marqo_b200 import model_registry as R

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available(), reason="needs an H100 (sm_90a)")]

NONE, CAUSAL, KEYLEN = 0, 1, 2
MASK_NAME = {NONE: "none", CAUSAL: "causal", KEYLEN: "keylen"}
MMA_S = [16, 77, 127]                        # the mma.sync kernel
WGMMA_S = [128, 129, 257, 385, 513, 1024]    # the wgmma kernel
EDGES = (1, 63, 64, 65, 127, 128, 129, 255, 256, 257)
H = 3                                        # heads of the bitwise cases
SMAX = 1024                                  # relative-bias table of the bitwise cases: any S here fits
HUGE_QK, HUGE_V = 1e30, 3e38                 # finite in bf16; q k of two of them overflows fp32
NAN = float("nan")


@pytest.fixture(scope="module")
def sm_count(gpu_required):
    return torch.cuda.get_device_properties(0).multi_processor_count


# ----------------------------------------------------------------------------------------------------- helpers
def _attention(qkv, B, S, Hn, mask=NONE, kv_len=None, bias=None, out=None):
    """b200_debug_attention on device buffers and the current stream: qkv bf16 [B * S, 3W] -> out bf16 [B * S, W].
    A fresh out starts as NaN, so an element the kernel does not write cannot pass as a result.  bias: fp32
    [Hn, 2 * smax - 1] host array, in natural-log units (the library scales it by log2(e))."""
    W = qkv.shape[1] // 3
    if out is None:
        out = torch.full((B * S, W), NAN, dtype=torch.bfloat16, device="cuda")
    kl = None if kv_len is None else torch.tensor(kv_len, dtype=torch.int32, device="cuda")
    rb, smax = None, 0
    if bias is not None:
        rb = np.ascontiguousarray(bias, np.float32)
        smax = (rb.shape[1] + 1) // 2
    N.check(N.load().b200_debug_attention(0, qkv.data_ptr(), B, S, W, Hn, mask, None if kl is None else kl.data_ptr(),
                                          None if rb is None else rb.ctypes.data_as(C.c_void_p), smax, out.data_ptr(),
                                          torch.cuda.current_stream().cuda_stream))
    return out


def _map_attention(q, kv, B, S, Hn):
    """b200_debug_map_attention on device buffers: q fp32 [W] (shared) or [B, W], kv bf16 [B * S, 2W] -> bf16 [B, W]."""
    W = q.shape[-1]
    out = torch.full((B, W), NAN, dtype=torch.bfloat16, device="cuda")
    N.check(N.load().b200_debug_map_attention(0, q.data_ptr(), 0 if q.dim() == 1 else W, kv.data_ptr(), B, S, W, Hn,
                                              out.data_ptr(), torch.cuda.current_stream().cuda_stream))
    return out


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _qkv(B, S, Hn, hd, seed):
    """Gaussian packed qkv, bf16 [B * S, 3 * Hn * hd]."""
    return torch.randn(B * S, 3 * Hn * hd, generator=_gen(seed), device="cuda").to(torch.bfloat16)


def _bias(Hn, smax, seed, scale=20.0):
    g = np.random.default_rng(seed)
    return g.uniform(-scale, scale, (Hn, 2 * smax - 1)).astype(np.float32)


def _huge(shape, value, seed):
    """+-value with random signs, bf16."""
    sign = torch.randint(0, 2, shape, generator=_gen(seed), device="cuda") * 2 - 1
    return (sign * value).to(torch.bfloat16)


def _assert_bits(got, want, what):
    g, w = got.contiguous().view(torch.int16), want.contiguous().view(torch.int16)
    diff = g != w
    if bool(diff.any()):
        idx = tuple(diff.nonzero()[0].tolist())
        pytest.fail(f"{what}: {int(diff.sum())} of {diff.numel()} elements differ, first at {idx}: "
                    f"{float(got[idx])!r} vs {float(want[idx])!r}")


def _edges(S):
    """The key lengths / query rows where tiles end, that fit in S, with S - 1 and S."""
    return sorted({e for e in EDGES if e <= S} | {S - 1, S} - {0})


def _cases(with_bias=True):
    """(S, hd, bias) for both head dims, plus MPNet's relative bias (head_dim 64 only)."""
    out = []
    for S in MMA_S + WGMMA_S:
        for hd, bias in [(32, False), (64, False)] + ([(64, True)] if with_bias else []):
            out.append(pytest.param(S, hd, bias, id=f"S{S}-hd{hd}" + ("-bias" if bias else "")))
    return out


# ---------------------------------------------------------------------------- A. properties that hold bit for bit
@pytest.mark.parametrize("S,hd,bias", _cases())
def test_masked_keys_have_no_effect(gpu_required, S, hd, bias):
    """One copy of the sequence per key length L: K and V of tokens >= L overwritten with huge finite values give
    bitwise the output of those tokens zeroed, in every row (the rows >= L included)."""
    Ls = _edges(S)
    B = len(Ls)
    seq = _qkv(1, S, H, hd, seed=S * 7 + hd + bias).view(1, S, 3, H * hd)
    zeroed, huge = seq.repeat(B, 1, 1, 1), seq.repeat(B, 1, 1, 1)
    for b, L in enumerate(Ls):
        zeroed[b, L:, 1:] = 0
        huge[b, L:, 1] = _huge((S - L, H * hd), HUGE_QK, seed=b)
        huge[b, L:, 2] = _huge((S - L, H * hd), HUGE_V, seed=b + 1000)
    tb = _bias(H, SMAX, seed=S) if bias else None
    want = _attention(zeroed.view(B * S, -1), B, S, H, KEYLEN, Ls, tb)
    got = _attention(huge.view(B * S, -1), B, S, H, KEYLEN, Ls, tb)
    assert bool(torch.isfinite(want).all())
    _assert_bits(got, want, "huge masked keys vs zeroed masked keys")


@pytest.mark.parametrize("S,hd,bias", _cases())
def test_masked_equals_truncated(gpu_required, S, hd, bias):
    """Rows < L of (S, kv_len = L) equal the sequence cut to its first L tokens with no mask, when S and L take the
    same kernel; when L < 128 <= S, the cut is to 128 tokens with kv_len = L.  With the bias both sides use the
    key-length mask (the only mask the bias runs with) and the same table."""
    Ls = _edges(S)
    B = len(Ls)
    seq = _qkv(1, S, H, hd, seed=S * 11 + hd + bias)
    tb = _bias(H, SMAX, seed=S + 1) if bias else None
    masked = _attention(seq.repeat(B, 1), B, S, H, KEYLEN, Ls, tb).view(B, S, -1)
    for b, L in enumerate(Ls):
        cut, cut_len = (L, L) if (L >= 128) == (S >= 128) else (128, L)
        part = seq[:cut].contiguous()
        if bias:
            short = _attention(part, 1, cut, H, KEYLEN, [cut_len], tb)
        elif cut_len == cut:
            short = _attention(part, 1, cut, H, NONE)
        else:
            short = _attention(part, 1, cut, H, KEYLEN, [cut_len])
        _assert_bits(masked[b, :L], short[:L], f"kv_len {L} vs the first {cut} tokens with {cut_len} keys")


@pytest.mark.parametrize("S,hd,bias", _cases())
def test_key_length_is_clamped(gpu_required, S, hd, bias):
    """kv_len S + 1 and 2^31 - 1 give bitwise the output of kv_len = S, which equals MASK_NONE; kv_len 0 and -5 give
    rows of +0."""
    lens = [S, S + 1, 2**31 - 1, 0, -5]
    B = len(lens)
    seq = _qkv(1, S, H, hd, seed=S * 13 + hd + bias)
    tb = _bias(H, SMAX, seed=S + 2) if bias else None
    got = _attention(seq.repeat(B, 1), B, S, H, KEYLEN, lens, tb).view(B, S, -1)
    _assert_bits(got[1], got[0], "kv_len S + 1 vs S")
    _assert_bits(got[2], got[0], "kv_len 2^31 - 1 vs S")
    if not bias:
        _assert_bits(_attention(seq, 1, S, H, NONE), got[0], "MASK_NONE vs kv_len S")
    _assert_bits(got[3:], torch.zeros_like(got[3:]), "rows without keys (kv_len 0, -5)")


@pytest.mark.parametrize("S,hd,bias", _cases(with_bias=False))
def test_causal_row_equals_key_length(gpu_required, S, hd, bias):
    """Row i under MASK_CAUSAL equals row i of MASK_KEYLEN with kv_len = i + 1, at the rows where tiles end."""
    rows = sorted({i for e in _edges(S) for i in (e - 1, e) if 0 <= i < S} | {0})
    seq = _qkv(1, S, H, hd, seed=S * 17 + hd)
    causal = _attention(seq, 1, S, H, CAUSAL)
    keylen = _attention(seq.repeat(len(rows), 1), len(rows), S, H, KEYLEN, [i + 1 for i in rows]).view(len(rows), S, -1)
    for b, i in enumerate(rows):
        _assert_bits(causal[i], keylen[b, i], f"causal row {i} vs kv_len {i + 1}")


def _mask_cases(seqs):
    """(S, hd, mask, bias): every mask at both head dims, and the key-length mask with the bias at head_dim 64."""
    out = []
    for S in seqs:
        for hd in (32, 64):
            for mask, bias in [(NONE, False), (CAUSAL, False), (KEYLEN, False)] + ([(KEYLEN, True)] if hd == 64 else []):
                out.append(pytest.param(S, hd, mask, bias, id=f"S{S}-hd{hd}-{MASK_NAME[mask]}" + ("-bias" if bias else "")))
    return out


# not multiples of 128: the last K / V tile runs into the next sequence
@pytest.mark.parametrize("S,hd,mask,bias", _mask_cases([16, 77, 127, 129, 257, 385, 513]))
def test_sequences_are_isolated(gpu_required, S, hd, mask, bias):
    """Each sequence of a batch of 3 random ones equals its run alone (B = 1), and sequence 1 between two neighbours
    of huge finite values does too.  The key lengths are S, so the mask that keeps the next sequence out is the
    sequence's end."""
    seqs = [_qkv(1, S, H, hd, seed=S * 19 + hd + 3 * b + mask + bias) for b in range(3)]
    tb = _bias(H, SMAX, seed=S + 3) if bias else None
    kl = (lambda n: [S] * n) if mask == KEYLEN else (lambda n: None)
    alone = [_attention(s, 1, S, H, mask, kl(1), tb) for s in seqs]
    batch = _attention(torch.cat(seqs), 3, S, H, mask, kl(3), tb).view(3, S, -1)
    for b in range(3):
        _assert_bits(batch[b], alone[b], f"sequence {b} of a batch vs alone")
    W = H * hd
    big = [torch.cat([_huge((S, 2 * W), HUGE_QK, seed=10 + b), _huge((S, W), HUGE_V, seed=20 + b)], 1) for b in (0, 2)]
    fenced = _attention(torch.cat([big[0], seqs[1], big[1]]), 3, S, H, mask, kl(3), tb).view(3, S, -1)
    _assert_bits(fenced[1], alone[1], "sequence between huge neighbours vs alone")


@pytest.mark.parametrize("S,hd,mask,bias", _mask_cases([77, 257]))
def test_heads_are_independent(gpu_required, S, hd, mask, bias):
    """Permuting the heads of Q, K and V (and of the bias table) permutes the output heads, bitwise."""
    Hn, B = 4, 2
    perm = [2, 0, 3, 1]
    qkv = _qkv(B, S, Hn, hd, seed=S * 23 + hd + mask)
    lens = [S, S // 2 + 1] if mask == KEYLEN else None
    tb = _bias(Hn, SMAX, seed=S + 4) if bias else None
    got = _attention(qkv, B, S, Hn, mask, lens, tb).view(B * S, Hn, hd)
    pq = qkv.view(B * S, 3, Hn, hd)[:, :, perm].reshape(B * S, -1).contiguous()
    pb = None if tb is None else tb[perm]
    permuted = _attention(pq, B, S, Hn, mask, lens, pb).view(B * S, Hn, hd)
    _assert_bits(permuted, got[:, perm], "permuted heads")


@pytest.mark.parametrize("mask", [NONE, CAUSAL, KEYLEN], ids=["none", "causal", "keylen"])
@pytest.mark.parametrize("hd", [32, 64])
def test_batch_at_the_grid_limit(gpu_required, hd, mask):
    """B = 65535 sequences of one token (gridDim.z at its limit): each output row is its V row, bit for bit (p = 1,
    P = 1, row sum 1), up to the last sequence; with the key-length mask, every third sequence has no key and is +0."""
    B = 65535
    qkv = _qkv(B, 1, 1, hd, seed=hd + mask)
    lens = [0 if b % 3 == 1 else 1 for b in range(B)] if mask == KEYLEN else None
    got = _attention(qkv, B, 1, 1, mask, lens)
    want = qkv[:, 2 * hd:].clone()
    if lens is not None:
        want[1::3] = 0
    _assert_bits(got, want, "one-token sequences")
    _assert_bits(got[-1], want[-1], "the last sequence")


# -------------------------------------------------------------------------- B. every output element, nothing else
GUARD_ROWS = 64
GUARD_BITS = 0x3F81   # bf16 1.0078125: not NaN, not a value the kernel writes into a guard by chance


# S % 64 != 0: the last query block is partial
@pytest.mark.parametrize("S,hd,mask,bias", _mask_cases([16, 77, 127, 129, 197, 257, 1000]))
def test_output_coverage_and_containment(gpu_required, S, hd, mask, bias):
    """out sits between guard rows of a fixed bit pattern in a buffer otherwise filled with NaN: afterwards every
    element of out is finite, the guards are unchanged, and the sequences with kv_len <= 0 are exactly 0."""
    B, W = 4, H * hd
    lens = [S, 0, S // 2 + 1, -3] if mask == KEYLEN else None
    qkv = _qkv(B, S, H, hd, seed=S * 29 + hd + mask)
    buf = torch.full((GUARD_ROWS + B * S + GUARD_ROWS, W), NAN, dtype=torch.bfloat16, device="cuda")
    guard = torch.full((GUARD_ROWS, W), GUARD_BITS, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    buf[:GUARD_ROWS] = guard
    buf[-GUARD_ROWS:] = guard
    out = buf[GUARD_ROWS:GUARD_ROWS + B * S]
    assert out.is_contiguous()
    _attention(qkv, B, S, H, mask, lens, _bias(H, SMAX, seed=S) if bias else None, out=out)
    torch.cuda.synchronize()
    bad = ~torch.isfinite(out)
    assert not bool(bad.any()), f"{int(bad.sum())} output elements not written (still NaN), first at " \
                                f"{tuple(bad.nonzero()[0].tolist())}"
    _assert_bits(buf[:GUARD_ROWS], guard, "guard rows before out")
    _assert_bits(buf[-GUARD_ROWS:], guard, "guard rows after out")
    if lens is not None:
        o = out.view(B, S, W)
        _assert_bits(o[1], torch.zeros_like(o[1]), "kv_len 0")
        _assert_bits(o[3], torch.zeros_like(o[3]), "kv_len -3")


# ------------------------------------------------------------------------- C. error bound at every served shape
def _bound(s, a, vv, keep, bias_log2, hd, c, nkb, S, p_rounded):
    """Per-element bound on |kernel - fp64 softmax attention| for one batch of rows.

    Inputs, fp64, over the keys of each row: s the exact score q.k of the bf16 inputs, a = sum_i |q_i k_i|, vv the
    values, keep the unmasked keys, bias_log2 the bias in log2 units (or None), c = log2(e) / sqrt(hd) exactly, nkb the
    number of key blocks the row's CTA runs.  With x_j = c s_j + bias_j the exact log2-domain logits, w_j their
    softmax and ref = sum_j w_j v_j:

        |got - ref| <= 2^-8 |ref| + (1 + 2^-7) (u_P + 2 eps + (3 S / 4 + 8) 2^-24) sum_j w_j |v_j|

    Derivation.  The kernel computes o = bf16( (sum_j P_j v_j) / (sum_j p_j) ) with p_j = w_j K (1 + d_j) for one
    common K (the running maximum it subtracts cancels between numerator and denominator) and P_j = bf16(p_j) =
    p_j (1 + b_j), |b_j| <= u_P = 2^-8 (round to nearest).  Then

        o_pre - ref = sum_j w_j v_j [(1 + d_j)(1 + b_j) / (1 + dbar) - 1],   dbar = sum_j w_j d_j,

    which is at most (u_P + 2 eps) sum_j w_j |v_j| to first order when |d_j| <= eps.  eps collects, in log2 units
    times ln 2 (a logit error e changes p by a factor 2^e = 1 + ln2 e):
      - the score from the tensor core: hd exact products summed in fp32, each group of four products added exactly
        and truncated once (the H100's behaviour, test_score_bound_gpu.py), at most hd 2^-23 a_j, times c;
      - the fp32 scale c (3 roundings of 2^-24 for head_dim 32), the product s c, the bias scaled by log2(e) in fp32
        and its addition: 2^-21 X, X = max_j (|c s_j| + |bias_j|);
      - the subtraction of the maximum, 2^-24 |x_j - m| <= 2^-23 X, and for each of the nkb rescales the subtraction
        old - new (2^-23 X);
      - exp2f (2 ulp, 2^-22) for p and for each rescale, and the rounding of o *= corr and row_sum *= corr (2^-23);
    which gives eps = ln2 (c hd 2^-23 max_j a_j + (nkb + 4) 2^-22 X) + (nkb + 1) 2^-21.  The (3 S / 4 + 8) 2^-24 term
    covers the fp32 sums over the L <= S kept keys: the row sum of the unrounded p (a thread adds at most L / 4 + 2
    of them, then 2 quad additions), the P V sum on the tensor core (one truncation of 2^-23 per group of four keys,
    at most L / 4 + 1 groups hold a kept key; a group of exact zeros adds exactly) and 1 / row_sum and o * inv.
    The bf16 output rounding adds 2^-8 |o_pre| <= 2^-8 |ref| + 2^-8 |o_pre - ref|.  The factor 1 + 2^-7 covers that
    last term and every second-order product above (each below 2^-16 + 2^-7 eps).  p below fp32's normal range loses
    relative precision; such a key weighs less than 2^-126 and is far inside the 2^-24 term.  map_attention keeps P
    in fp32 (u_P = 0); its fp32 logits (64 fused multiply-adds of the fp32 query), its single maximum and its fp32
    sums (S / 4 + S / 128 + 12 roundings) fit the same eps and 2^-24 terms."""
    x = c * s
    X = (c * s).abs()
    if bias_log2 is not None:
        x = x + bias_log2
        X = X + bias_log2.abs()
    x = x.masked_fill(~keep, float("-inf"))
    w = torch.softmax(x * math.log(2.0), dim=-1)
    ref = w @ vv
    wabs = w @ vv.abs()
    Xm = X.masked_fill(~keep, 0).amax(-1, keepdim=True)
    Am = a.masked_fill(~keep, 0).amax(-1, keepdim=True)
    eps = math.log(2.0) * (c * hd * 2.0**-23 * Am + (nkb + 4) * 2.0**-22 * Xm) + (nkb + 1) * 2.0**-21
    u_p = 2.0**-8 if p_rounded else 0.0
    return ref, 2.0**-8 * ref.abs() + (1 + 2.0**-7) * (u_p + 2 * eps + (0.75 * S + 8) * 2.0**-24) * wabs


def _within_bound(got, q, k, v, keep, bias_log2, hd, c, nkb, S, p_rounded):
    """Fails on the first element of got [B, Hn, rows, hd] over _bound, and returns the worst ratio error / bound.
    q [B, Hn, rows, hd], k, v [B, Hn, S, hd] hold the bf16 inputs (q fp32 for map_attention), keep [B, 1, rows, S],
    nkb a number or [B, 1, rows, 1].  The fp64 scores are formed a few sequences at a time: a whole batch of them
    would take tens of GB."""
    worst = 0.0
    chunk = max(1, 2**25 // (q.shape[1] * q.shape[2] * S))
    for b0 in range(0, got.shape[0], chunk):
        sl = slice(b0, b0 + chunk)
        qc, kc = q[sl].double(), k[sl].double()
        ref, bound = _bound(qc @ kc.transpose(-1, -2), qc.abs() @ kc.abs().transpose(-1, -2), v[sl].double(),
                            keep[sl], bias_log2, hd, c, nkb[sl] if torch.is_tensor(nkb) else nkb, S, p_rounded)
        err = (got[sl] - ref).abs()
        over = err > bound
        if bool(over.any()):
            i = tuple(over.nonzero()[0].tolist())
            pytest.fail(f"{int(over.sum())} elements over the bound, first at [b, h, row, col] "
                        f"{(b0 + i[0],) + i[1:]}: got {float(got[sl][i])!r}, ref {float(ref[i])!r}, "
                        f"bound {float(bound[i]):.3g}")
        worst = max(worst, float((err / bound).max()))
    return worst


RESIDENT_CTAS_PER_SM = 32   # the most CTAs an H100 SM holds at once, whatever a kernel's registers and shared memory


def _over_one_wave(sm_count, ctas_per_item):
    """Sequences (or images) whose grid is larger than one wave: more CTAs than all the SMs can hold at once."""
    return RESIDENT_CTAS_PER_SM * sm_count // ctas_per_item + 1


def _served_attention():
    """{(S, H, hd, mask, bias): tower} for every attention of every entry find_model reaches.  Vision towers run
    without a mask at their token count; CLIP text towers (of the ViT, ResNet and ConvNeXt models) causal at 77;
    SigLIP text without a mask at 64.  The BERT, XLM-R and MPNet towers run with key lengths, MPNet with its relative
    bias, at S = the longest text of the batch (texts are padded to it), so at any S up to their token limit: here
    at the tile edges of both kernels (16, 63, 64, 65, 77 and 127 on mma.sync; 129, 257 and 512, the longest any of
    them takes, on wgmma) and at the token limit."""
    shapes = {}
    tables = (R.MODELS, R.MPNET_MODELS, R.SIGLIP_MODELS, R.XLMR_MODELS, R.RESNET_MODELS, R.CONVNEXT_MODELS)
    for table in tables:
        for entry in table.values():
            a = entry["arch"]
            kind = a.get("kind")
            if kind == "siglip":
                v, t = a["vision"], a["text"]
                shapes.setdefault(((v["image_size"] // v["patch"]) ** 2, v["heads"], v["width"] // v["heads"], NONE,
                                   False), "siglip-vision")
                shapes.setdefault((t["ctx"], t["heads"], t["width"] // t["heads"], NONE, False), "siglip-text")
            elif kind in ("clip_resnet", "clip_convnext"):
                shapes.setdefault((a["ctx"], a["heads"], a["width"] // a["heads"], CAUSAL, False), "clip-text")
            elif "vision" in a:
                v, t = a["vision"], a["text"]
                shapes.setdefault(((v["image_size"] // v["patch"]) ** 2 + 1, v["heads"], v["width"] // v["heads"],
                                   NONE, False), "clip-vision")
                shapes.setdefault((t["ctx"], t["heads"], t["width"] // t["heads"], CAUSAL, False), "clip-text")
            else:
                for S in {16, 63, 64, 65, 77, 127, 129, 257, 512, entry["tokens"]}:
                    shapes.setdefault((S, a["heads"], a["width"] // a["heads"], KEYLEN, kind == "mpnet"),
                                      kind or "bert")
    return shapes


def test_served_attention_shapes():
    """The enumeration reaches every attention shape the registry serves today: a table it stops reaching shows here."""
    s = _served_attention()
    assert {(S, h, m) for (S, h, hd, m, b) in s if hd == 64 and m == NONE} >= {
        (50, 12, NONE), (197, 12, NONE), (257, 16, NONE), (196, 12, NONE), (256, 12, NONE), (576, 12, NONE),
        (1024, 12, NONE), (256, 16, NONE), (576, 16, NONE), (64, 12, NONE), (64, 16, NONE)}
    assert {h for (S, h, hd, m, b) in s if m == CAUSAL} == {8, 10, 12, 16}
    short = {16, 63, 64, 65, 77, 127}
    for hd in (32, 64):
        assert {S for (S, h, d, m, b) in s if d == hd and m == KEYLEN and not b} >= short | {129, 257, 512}
    assert {S for (S, h, hd, m, b) in s if b} == short | {128, 129, 257, 512}


# Floors of the adversarial families: half the smallest worst ratio measured on an H100 over the family's shapes (the
# range of worst ratios over those shapes follows each entry).  Gaussian inputs (0.27 .. 0.90 for attention, 0.78 ..
# 0.93 for map_attention) have no floor; a single key is exact.
FLOORS = {
    "peaked": 0.36,              # 0.730 .. 0.872
    "v_offset": 0.17,            # 0.346 .. 0.568
    "dominant_last": 0.24,       # 0.480 .. 0.911
    "bias20": 0.41,              # 0.838 .. 0.900
    "map_peaked": 0.39,          # 0.793 .. 0.827
    "map_v_offset": 0.30,        # 0.617 .. 0.629
    "map_dominant_last": 0.46,   # 0.939 .. 0.955
}


def _bound_cases():
    cases = []
    for (S, Hn, hd, mask, bias), tower in sorted(_served_attention().items()):
        fams = ["gaussian", "peaked", "v_offset"]
        if S in (65, 129, 197, 257):
            fams.append("dominant_last")
        if mask == KEYLEN:
            fams.append("single_key")
        if bias:
            fams.append("bias20")
        for f in fams:
            cases.append(pytest.param(S, Hn, hd, mask, bias, f,
                                      id=f"{f}-{tower}-S{S}-H{Hn}-hd{hd}-{MASK_NAME[mask]}" + ("-bias" if bias else "")))
    return cases


def _family_inputs(f, B, S, Hn, hd, seed):
    """qkv fp32 (bf16 values) [B, S, 3, Hn, hd] of family f."""
    g = _gen(seed)
    x = torch.randn(B, S, 3, Hn, hd, generator=g, device="cuda")
    if f == "peaked":
        x[:, :, :2] *= 3.0                     # score std 9
    elif f == "v_offset":
        x[:, :, 2] += 100.0
    elif f == "dominant_last":                  # the last key, alone in its tile at 65, 129 and 257, takes most rows
        u = torch.randn(B, 1, Hn, hd, generator=g, device="cuda")
        x[:, :, 0] += u
        x[:, S - 1, 1] = u[:, 0] * (9.0 / math.sqrt(hd))
    return x.to(torch.bfloat16).float()


def _nkb(S, mask, lens):
    """Key blocks of each (sequence, query row)'s CTA (attention.cuh: key_range) -> [B, 1, S, 1]."""
    bkv = 128 if S >= 128 else 64
    q0 = (torch.arange(S, device="cuda") // 64) * 64
    length = torch.tensor(lens, device="cuda").clamp(0, S)[:, None]
    kend = torch.minimum(length, q0[None] + 64) if mask == CAUSAL else length.expand(-1, S)
    return ((kend + bkv - 1) // bkv).double()[:, None, :, None]


@pytest.mark.parametrize("S,Hn,hd,mask,bias,family", _bound_cases())
def test_error_within_bound(sm_count, S, Hn, hd, mask, bias, family):
    B = _over_one_wave(sm_count, -(-S // 64) * Hn)
    W = Hn * hd
    x = _family_inputs(family, B, S, Hn, hd, seed=S * 31 + Hn * 7 + hd + mask + len(family))
    g = torch.Generator().manual_seed(S + Hn)
    lens = None
    if mask == KEYLEN:
        lens = [1] * B if family == "single_key" else torch.randint(1, S + 1, (B,), generator=g).tolist()
        if family != "single_key":
            lens[0] = S
    tb = None
    if bias:
        tb = _bias(Hn, 512, seed=S, scale=20.0 if family == "bias20" else 2.0)
    got = _attention(x.reshape(B * S, 3 * W).to(torch.bfloat16), B, S, Hn, mask, lens, tb)
    got = got.view(B, S, Hn, hd).permute(0, 2, 1, 3).double()          # [B, Hn, S, hd]
    q, k, v = x.permute(2, 0, 3, 1, 4)                                  # [B, Hn, S, hd] each
    key = torch.arange(S, device="cuda")
    length = torch.tensor(lens if lens is not None else [S] * B, device="cuda").clamp(0, S)
    keep = (key[None, None, None, :] < length[:, None, None, None]).expand(B, 1, S, S)
    if mask == CAUSAL:
        keep = keep & (key[None, None, None, :] <= key[None, None, :, None])
    bias_log2 = None
    if tb is not None:
        rel = (key[None, :] - key[:, None] + 512 - 1)
        bias_log2 = torch.from_numpy(tb).cuda().double()[:, rel][None] * math.log2(math.e)
    c = math.log2(math.e) / math.sqrt(hd)
    assert bool(torch.isfinite(got).all())
    if family == "single_key":   # one key: p = 1, P = 1, row sum 1, so every row is its sequence's first V row
        assert torch.equal(got, v[:, :, :1].double().expand_as(got)), "kv_len 1: an output row is not its first V row"
    ratio = _within_bound(got, q, k, v, keep, bias_log2, hd, c, _nkb(S, mask, lens or [S] * B), S, True)
    print(f"\n[attention bound] {family} S={S} H={Hn} hd={hd} {MASK_NAME[mask]}{' bias' if bias else ''} B={B}: "
          f"worst ratio {ratio:.4f}")
    floor = FLOORS.get(family)
    if floor is not None:
        assert ratio >= floor, f"{family}: worst ratio {ratio:.4g} no longer reaches {floor}"


# ------------------------------------------------------------------------------------------- D. map_attention
def _served_map():
    """{(S, H, per-image query): tower}: the SigLIP MAP heads (one shared query over the vision tokens) and the
    ResNet attention pools (the mean token as each image's query, over the 7 x 7 grid and the mean)."""
    shapes = {}
    for e in R.SIGLIP_MODELS.values():
        v = e["arch"]["vision"]
        shapes.setdefault(((v["image_size"] // v["patch"]) ** 2, v["heads"], False), "siglip-map")
    for e in R.RESNET_MODELS.values():
        r = e["arch"]["resnet"]
        shapes.setdefault(((r["image_size"] // 32) ** 2 + 1, r["heads"], True), "resnet-attnpool")
    return shapes


def _map_cases():
    cases = []
    for (S, Hn, per_image), tower in sorted(_served_map().items()):
        for f in ("gaussian", "peaked", "v_offset", "dominant_last"):
            cases.append(pytest.param(S, Hn, per_image, f, id=f"{f}-{tower}-S{S}-H{Hn}"))
    return cases


def _map_inputs(f, B, S, Hn, per_image, seed):
    """(q fp32 [W] or [B, W], kv bf16 values as fp32 [B, S, 2, Hn, 64]) of family f."""
    g = _gen(seed)
    q = torch.randn(B if per_image else 1, Hn, 64, generator=g, device="cuda")
    kv = torch.randn(B, S, 2, Hn, 64, generator=g, device="cuda")
    if f == "peaked":
        q *= 3.0
        kv[:, :, 0] *= 3.0
    elif f == "v_offset":
        kv[:, :, 1] += 100.0
    elif f == "dominant_last":
        kv[:, S - 1, 0] = q.expand(B, Hn, 64) * (72.0 / (q * q).sum(-1, keepdim=True))   # logit q.k / 8 = 9
    q = q.reshape(B if per_image else 1, Hn * 64)
    return (q if per_image else q[0]).contiguous(), kv.to(torch.bfloat16).float()


@pytest.mark.parametrize("S,Hn,per_image,family", _map_cases())
def test_map_attention_within_bound(sm_count, S, Hn, per_image, family):
    B = _over_one_wave(sm_count, Hn)
    W = Hn * 64
    q, kv = _map_inputs(family, B, S, Hn, per_image, seed=S * 37 + Hn + len(family))
    got = _map_attention(q, kv.reshape(B * S, 2 * W).to(torch.bfloat16), B, S, Hn).view(B, Hn, 1, 64).double()
    qd = q.view(-1, Hn, 1, 64).expand(B, Hn, 1, 64)
    k, v = kv.permute(2, 0, 3, 1, 4)                                     # [B, Hn, S, 64]
    keep = torch.ones(B, 1, 1, S, dtype=torch.bool, device="cuda")
    assert bool(torch.isfinite(got).all())
    ratio = _within_bound(got, qd, k, v, keep, None, 64, math.log2(math.e) / 8.0, 1, S, False)
    print(f"\n[map bound] {family} S={S} H={Hn} {'per-image' if per_image else 'shared'} query B={B}: "
          f"worst ratio {ratio:.4f}")
    floor = FLOORS.get("map_" + family)
    if floor is not None:
        assert ratio >= floor, f"map {family}: worst ratio {ratio:.4g} no longer reaches {floor}"


@pytest.mark.parametrize("S,Hn,per_image", [pytest.param(S, Hn, p, id=f"{t}-S{S}-H{Hn}")
                                            for (S, Hn, p), t in sorted(_served_map().items())])
def test_map_attention_images_are_isolated(gpu_required, S, Hn, per_image):
    """Image 1 of three gives bitwise its output alone, with random neighbours and with neighbours of huge values."""
    W = Hn * 64
    q, kv = _map_inputs("gaussian", 3, S, Hn, per_image, seed=S + Hn)
    kv = kv.to(torch.bfloat16)
    q1 = q[1:2].contiguous() if per_image else q
    alone = _map_attention(q1, kv[1].reshape(S, 2 * W).contiguous(), 1, S, Hn)
    batch = _map_attention(q, kv.reshape(3 * S, 2 * W), 3, S, Hn)
    _assert_bits(batch[1], alone[0], "image 1 of a batch vs alone")
    big = kv.clone()
    big[0, :, 0] = _huge((S, Hn, 64), HUGE_QK, seed=1)
    big[2, :, 0] = _huge((S, Hn, 64), HUGE_QK, seed=2)
    big[0, :, 1] = _huge((S, Hn, 64), HUGE_V, seed=3)
    big[2, :, 1] = _huge((S, Hn, 64), HUGE_V, seed=4)
    fenced = _map_attention(q, big.reshape(3 * S, 2 * W), 3, S, Hn)
    _assert_bits(fenced[1], alone[0], "image 1 between huge neighbours vs alone")
