"""Kernel-level tests of the encoders' embedding, pooling and head kernels (kernels.cuh) against plain torch references
written from the documented semantics, in fp64 where the operation is not exact.  Each kernel runs through its
b200_debug_* hook, which calls exactly the kernels:: function the model calls.

The kernels are memory-bound and simple, so the bars are strict: copies and sums of two fp32 values are compared bit
for bit, bf16 outputs to within one bf16 ulp of the fp64 value, and reductions at a tolerance derived from their fp32
arithmetic.  The end-to-end tower tests compare pooled vectors at a cosine of 1 - 1e-3, which cannot see one token
missing from a mean or a position id off by one."""
import math

import pytest
import torch

from _checks import bf16
from marqo_b200 import _native as N

pytestmark = pytest.mark.gpu

F = torch.nn.functional
CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


def _assert_within_bf16_ulp(got: torch.Tensor, ref: torch.Tensor) -> None:
    """|got - ref| <= one bf16 ulp at |ref| (the spacing of bf16 values there: 2^(e - 7) for |ref| in [2^e, 2^(e+1))),
    and got == 0 where ref == 0.  A correctly rounded result is within half an ulp; the other half leaves room for an
    fp32 intermediate that sits next to a rounding boundary."""
    ref = ref.double()
    ulp = torch.ldexp(torch.ones_like(ref), torch.frexp(ref).exponent - 8)
    tol = torch.where(ref == 0, torch.zeros_like(ref), ulp)
    err = (got.double() - ref).abs()
    bad = err > tol
    assert not bad.any(), (f"{int(bad.sum())} of {bad.numel()} values beyond one bf16 ulp; first at "
                           f"{tuple(bad.nonzero()[0].tolist())}: got {float(got.double()[bad][0])}, "
                           f"ref {float(ref[bad][0])}")


def _layer_norm64(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float) -> torch.Tensor:
    return F.layer_norm(x.double(), (x.shape[-1],), gamma.double(), beta.double(), eps)


def _ln_params(w: int, g: torch.Generator):
    return 1.0 + 0.1 * torch.randn(w, generator=g), 0.1 * torch.randn(w, generator=g)


# LayerNorm outputs here have |y| <~ 5.  The fp32 kernel's error is a few ulps of the mean, of the variance and of the
# output itself (~1e-6); 1e-5 leaves room, while a wrong row or position (an O(1) change) fails by orders of magnitude.
LN_TOL = dict(rtol=1e-5, atol=1e-5)


# ------------------------------------------------------------------------------------------------ clip_text_embed
def _text_ids(n: int, S: int, vocab: int, g: torch.Generator) -> torch.Tensor:
    """Rows that cycle through: the maximum id repeated (first at 3, again at 9 and S - 1), the maximum at position 0,
    the maximum at S - 1, and ids from a small range so that maxima tie at random places."""
    ids = torch.randint(0, vocab - 1, (n, S), generator=g, dtype=torch.int32)
    for b in range(n):
        kind = b % 4
        if kind == 0:
            ids[b] = torch.randint(0, vocab // 2, (S,), generator=g)
            for s in (3, 9, S - 1):
                if s < S:
                    ids[b, s] = vocab - 1
        elif kind == 1:
            ids[b, 0] = vocab - 1
        elif kind == 2:
            ids[b, S - 1] = vocab - 1
        else:
            ids[b] = torch.randint(0, 8, (S,), generator=g)
    return ids


@pytest.mark.parametrize("n,S,w", [(1, 77, 512), (3, 77, 768), (5, 64, 768), (9, 64, 1024), (257, 77, 512),
                                   (257, 64, 384)])
def test_clip_text_embed(gpu_required, n, S, w):
    """CLIP (S = 77) and SigLIP (S = 64) text: x = tok[ids] + pos[s] bit for bit (one fp32 add), eot = the first
    arg-max of each row (torch.argmax, which CLIP's text_global_pool uses)."""
    from marqo_b200.engine import debug_clip_text_embed
    g = torch.Generator().manual_seed(n * 100 + S + w)
    vocab = 1000
    tok = torch.randn(vocab, w, generator=g)
    pos = torch.randn(S, w, generator=g)
    ids = _text_ids(n, S, vocab, g)
    x, eot = debug_clip_text_embed(ids.numpy(), tok.numpy(), pos.numpy())
    ref = (tok[ids.long()] + pos[None]).reshape(n * S, w)
    assert torch.equal(torch.from_numpy(x), ref)
    want = ids.argmax(-1).to(torch.int32)
    assert torch.equal(torch.from_numpy(eot), want), (eot, want)
    assert want[:3].tolist() == [3, 0, S - 1][:n]


# ------------------------------------------------------------------------------------------------ bert_embed_ln
def _prefix_mask(n: int, S: int, g: torch.Generator) -> torch.Tensor:
    """Random key lengths in [1, S], with full rows and length-1 rows among them."""
    lens = torch.randint(1, S + 1, (n,), generator=g)
    lens[0] = S
    if n > 1:
        lens[1] = 1
    return (torch.arange(S)[None, :] < lens[:, None]).to(torch.int32)


@pytest.mark.parametrize("n,S,w,masked", [(1, 1, 384, False), (3, 512, 384, True), (5, 77, 768, True),
                                          (9, 128, 1024, False), (257, 16, 512, True), (2, 512, 1024, True)])
def test_bert_embed_ln(gpu_required, n, S, w, masked):
    """x = LN((word[ids] + type0) + pos[s]) at fp32 accuracy; h = x rounded to bf16 (round to nearest even) bit for
    bit; kv_len = mask.sum(1), or S without a mask.  The position is the token's place in its row, whatever the mask."""
    from marqo_b200.engine import debug_embed_ln
    g = torch.Generator().manual_seed(n * 1000 + S + w)
    vocab, max_pos, eps = 1000, 512, 1e-12
    word = 0.5 * torch.randn(vocab, w, generator=g)
    pos = 0.5 * torch.randn(max_pos, w, generator=g)
    type0 = 0.5 * torch.randn(w, generator=g)
    gamma, beta = _ln_params(w, g)
    ids = torch.randint(0, vocab, (n, S), generator=g, dtype=torch.int32)
    mask = _prefix_mask(n, S, g) if masked else None
    if masked and n > 2:
        mask[2, S // 3] = 0   # a hole: kv_len counts the ones, not the prefix
    x, h, kv_len = debug_embed_ln(ids.numpy(), None if mask is None else mask.numpy(), word.numpy(), pos.numpy(),
                                  type0.numpy(), gamma.numpy(), beta.numpy(), eps)
    x, h = torch.from_numpy(x), torch.from_numpy(h)
    e = (word[ids.long()].double() + type0.double()) + pos[:S].double()[None]
    ref = _layer_norm64(e, gamma, beta, eps).reshape(n * S, w)
    torch.testing.assert_close(x.double(), ref, **LN_TOL)
    assert torch.equal(h, bf16(x))
    want = mask.sum(1).to(torch.int32) if masked else torch.full((n,), S, dtype=torch.int32)
    assert torch.equal(torch.from_numpy(kv_len), want)


# ------------------------------------------------------------------------------------------------ roberta_embed_ln
PAD = 1   # XLM-R's and MPNet's pad id


def _roberta_ids(n: int, S: int, vocab: int, no_pads: bool, g: torch.Generator):
    """ids and mask with rows that cycle through: pads in the tail, pads inside the unmasked prefix (the position ids
    still skip them), a row of all pads (mask all zero) and a row without pads."""
    ids = torch.randint(PAD + 1, vocab, (n, S), generator=g, dtype=torch.int32)
    ids[:, 0] = 0   # <s>
    mask = torch.ones(n, S, dtype=torch.int32)
    if no_pads:
        return ids, mask
    for b in range(n):
        kind = b % 4
        L = int(torch.randint(max(1, S // 2), S + 1, (1,), generator=g))
        if kind in (0, 1):
            ids[b, L:] = PAD
            mask[b, L:] = 0
        if kind == 1:
            for s in (1, L // 2, L - 1):
                ids[b, s] = PAD   # inside the unmasked prefix: mask stays 1
        if kind == 2:
            ids[b] = PAD
            mask[b] = 0
    return ids, mask


def _hf_positions(ids: torch.Tensor, pad: int) -> torch.Tensor:
    """HF RoBERTa create_position_ids_from_input_ids: positions count the non-pad ids, from the ids and not the mask."""
    keep = (ids != pad).long()
    return torch.cumsum(keep, dim=1) * keep + pad


@pytest.mark.parametrize("n,S,w,type_row,no_pads", [
    (1, 512, 768, True, True),      # 512 tokens: positions reach row 513, the last of a 514-row table
    (2, 512, 1024, False, True),
    (3, 77, 384, False, False),
    (5, 128, 1024, True, False),
    (9, 40, 768, False, False),
    (257, 16, 512, True, False),
])
def test_roberta_embed_ln(gpu_required, n, S, w, type_row, no_pads):
    """x = LN(word[ids] (+ type0) + pos[p]) with HF's position ids p; type0 None is MPNet's kernel instantiation."""
    from marqo_b200.engine import debug_embed_ln
    g = torch.Generator().manual_seed(n * 1000 + S + w)
    vocab, eps = 1000, 1e-5
    pos_rows = 512 + PAD + 1
    word = 0.5 * torch.randn(vocab, w, generator=g)
    pos = 0.5 * torch.randn(pos_rows, w, generator=g)
    type0 = 0.5 * torch.randn(w, generator=g) if type_row else None
    gamma, beta = _ln_params(w, g)
    ids, mask = _roberta_ids(n, S, vocab, no_pads, g)
    p = _hf_positions(ids, PAD)
    try:
        from transformers.models.roberta.modeling_roberta import RobertaEmbeddings
        assert torch.equal(p, RobertaEmbeddings.create_position_ids_from_input_ids(ids.long(), PAD))
    except ImportError:
        pass
    if no_pads:
        assert int(p.max()) == PAD + S
    x, h, kv_len = debug_embed_ln(ids.numpy(), mask.numpy(), word.numpy(), pos.numpy(),
                                  None if type0 is None else type0.numpy(), gamma.numpy(), beta.numpy(), eps, pad=PAD)
    x, h = torch.from_numpy(x), torch.from_numpy(h)
    e = word[ids.long()].double()
    if type0 is not None:
        e = e + type0.double()
    e = e + pos.double()[p]
    ref = _layer_norm64(e, gamma, beta, eps).reshape(n * S, w)
    torch.testing.assert_close(x.double(), ref, **LN_TOL)
    assert torch.equal(h, bf16(x))
    assert torch.equal(torch.from_numpy(kv_len), mask.sum(1).to(torch.int32))


# ------------------------------------------------------------------------------------------------ clip_head
@pytest.mark.parametrize("normalize", [True, False])
@pytest.mark.parametrize("n,S,w,E,rows", [
    (1, 50, 768, 512, False),       # ViT image head: the class token, row 0
    (3, 77, 512, 512, True),        # CLIP text head: the EOT row
    (5, 77, 1024, 768, True),
    (9, 257, 768, 100, False),      # E not a multiple of 64: a partial column tile
    (257, 77, 1024, 1024, True),    # 257 images: a last CTA of one image
    (6, 20, 384, 100, True),
])
def test_clip_head(gpu_required, n, S, w, E, rows, normalize):
    """out = LN(x[b*S + row_in_seq[b]]) @ proj, then / |.| when normalize (no epsilon), in fp64.
    Tolerance: the projection sums w <= 1024 fp32 products into outputs of std ~1; each add rounds by at most half an
    ulp of a partial sum |.| < 2 (6e-8), under 1e-4 even if every rounding went the same way (the typical error is
    ~1e-6).  A row, column or K-slice out of place moves outputs by O(0.1..1).  Normalised outputs are ~sqrt(E)
    smaller, and so is the bound."""
    from marqo_b200.engine import debug_clip_head
    g = torch.Generator().manual_seed(n * 7 + S + w + E)
    eps = 1e-5
    x = torch.randn(n * S, w, generator=g) * 2 + 0.5
    gamma, beta = _ln_params(w, g)
    proj = torch.randn(w, E, generator=g) / math.sqrt(w)
    r = None
    if rows:
        r = torch.randint(0, S, (n,), generator=g, dtype=torch.int32)
        r[0] = S - 1
        if n > 1:
            r[1] = 0
    got = torch.from_numpy(debug_clip_head(x.numpy(), S, gamma.numpy(), beta.numpy(), eps, proj.numpy(),
                                           row_in_seq=None if r is None else r.numpy(), normalize=normalize))
    sel = torch.arange(n) * S + (0 if r is None else r.long())
    ref = _layer_norm64(x[sel], gamma, beta, eps) @ proj.double()
    if normalize:
        ref = ref / ref.norm(dim=-1, keepdim=True)
    torch.testing.assert_close(got.double(), ref, rtol=0, atol=1e-4 / (math.sqrt(E) if normalize else 1.0))


# ------------------------------------------------------------------------------------------------ bert_head
@pytest.mark.parametrize("pool", [N.POOL_MEAN, N.POOL_CLS])
@pytest.mark.parametrize("normalize", [True, False])
@pytest.mark.parametrize("n,S,w", [(1, 1, 384), (3, 512, 768), (5, 77, 768), (9, 512, 1024), (257, 77, 384),
                                   (8, 77, 1024)])
def test_bert_head(gpu_required, n, S, w, pool, normalize):
    """Mean pooling over the first kv_len[b] rows (the reference's sum(h * mask) / sum(mask)) or the [CLS] row, then
    F.normalize (x / max(|x|, 1e-12)) when normalize.  kv_len > S counts S rows; kv_len 0 gives the reference's 0 / 0,
    a NaN row, under mean pooling and leaves CLS pooling alone.
    Tolerance: the mean adds <= 512 values of std 1 in fp32, partial sums |.| <~ 60, so at most 512 half-ulps of 60
    (1e-3) on the sum, 2e-6 on the mean; one token left out moves the mean by ~1/kv_len, far above 1e-5."""
    from marqo_b200.engine import debug_bert_head
    g = torch.Generator().manual_seed(n * 13 + S + w)
    x = torch.randn(n * S, w, generator=g)
    cycle = [1, 2, S - 1, S, S + 5, 0]
    kv_len = torch.tensor([cycle[b % len(cycle)] for b in range(n)], dtype=torch.int32)
    if n > len(cycle):
        kv_len[len(cycle):] = torch.randint(0, S + 1, (n - len(cycle),), generator=g, dtype=torch.int32)
    got = torch.from_numpy(debug_bert_head(x.numpy(), S, kv_len.numpy(), pool=pool, normalize=normalize))
    xs = x.double().view(n, S, w)
    if pool == N.POOL_CLS:
        ref = xs[:, 0]
    else:
        keep = (torch.arange(S)[None, :] < kv_len[:, None]).double()
        ref = (xs * keep[..., None]).sum(1) / keep.sum(1, keepdim=True)
    if normalize:
        ref = F.normalize(ref, dim=-1)
    assert torch.isnan(ref).any(dim=1).tolist() == [pool == N.POOL_MEAN and int(k) == 0 for k in kv_len]
    torch.testing.assert_close(got.double(), ref, rtol=1e-5, atol=1e-5, equal_nan=True)
    if pool == N.POOL_CLS and not normalize:
        assert torch.equal(got, x.view(n, S, w)[:, 0])


# ------------------------------------------------------------------------------------------------ l2_rows
@pytest.mark.parametrize("normalize", [True, False])
@pytest.mark.parametrize("n,E", [(3, 1), (5, 31), (9, 32), (257, 33), (1, 512), (257, 1024)])
def test_l2_rows(gpu_required, n, E, normalize):
    """out = src / |src| per row (no epsilon) or src unchanged.  Each output is one fp32 division by a norm whose sum
    of E squares loses at most ~(E/32 + 5) ulps (lane sums, then the warp's tree): < 4e-6 relative for E <= 1024."""
    from marqo_b200.engine import debug_l2_rows
    g = torch.Generator().manual_seed(n + E)
    src = torch.randn(n, E, generator=g) * 3
    got = torch.from_numpy(debug_l2_rows(src.numpy(), normalize=normalize))
    if not normalize:
        assert torch.equal(got, src)
        return
    ref = src.double() / src.double().norm(dim=-1, keepdim=True)
    torch.testing.assert_close(got.double(), ref, rtol=4e-6, atol=0)


# ------------------------------------------------------------------------------------------------ stem_im2col
def _stem_cols(chw: torch.Tensor) -> torch.Tensor:
    """conv1's im2col (3 x 3, stride 2, padding 1) of [n, 3, S, S] -> [n * (S/2)^2, 64], k = (3 ky + kx) * 3 + c,
    zero padding outside the image and in the columns k >= 27."""
    n, _, S, _ = chw.shape
    cols = F.unfold(chw, kernel_size=3, stride=2, padding=1)          # [n, c * 9 + tap, L]
    L = cols.shape[-1]
    assert L == (S // 2) ** 2
    cols = cols.view(n, 3, 9, L).permute(0, 3, 2, 1).reshape(n * L, 27)
    return F.pad(cols, (0, 64 - 27))


@pytest.mark.parametrize("u8", [False, True])
@pytest.mark.parametrize("n,S", [(3, 224), (5, 8), (9, 2), (257, 8)])
def test_stem_im2col(gpu_required, n, S, u8):
    """fp32 CHW input: every element is the bf16 of the gathered input, exactly, zero taps on all four borders and the
    zero columns k >= 27 included.  uint8 HWC input: within one bf16 ulp of (u8/255 - mean)/std in fp64 (the kernel
    normalises with a single fma on rounded constants, as the patch gather does)."""
    from marqo_b200.engine import debug_stem_im2col
    g = torch.Generator().manual_seed(n * 3 + S)
    if u8:
        img = torch.randint(0, 256, (n, S, S, 3), generator=g, dtype=torch.uint8)
        mean, std = torch.tensor(CLIP_MEAN, dtype=torch.float64), torch.tensor(CLIP_STD, dtype=torch.float64)
        chw = (img.permute(0, 3, 1, 2).double() / 255.0 - mean[None, :, None, None]) / std[None, :, None, None]
        got = torch.from_numpy(debug_stem_im2col(img.numpy(), CLIP_MEAN, CLIP_STD))
        _assert_within_bf16_ulp(got, _stem_cols(chw))
    else:
        chw = torch.randn(n, 3, S, S, generator=g)
        got = torch.from_numpy(debug_stem_im2col(chw.numpy()))
        assert torch.equal(got, bf16(_stem_cols(chw)))
    assert not got[:, 27:].any()


# ------------------------------------------------------------------------------------------------ avgpool2_nhwc
@pytest.mark.parametrize("n,H,W,C", [(2, 112, 112, 64), (3, 14, 14, 2048), (5, 2, 2, 8), (4, 2, 14, 64),
                                     (3, 112, 14, 8), (2, 14, 2, 2048)])
def test_avgpool2_nhwc(gpu_required, n, H, W, C):
    """AvgPool2d(2) on NHWC bf16: each output within one bf16 ulp of the fp64 mean of its four bf16 inputs."""
    from marqo_b200.engine import debug_avgpool2
    g = torch.Generator().manual_seed(n + H * W + C)
    x = bf16(torch.randn(n, H, W, C, generator=g))
    got = torch.from_numpy(debug_avgpool2(x.numpy()))
    ref = x.double().view(n, H // 2, 2, W // 2, 2, C).mean(dim=(2, 4))
    _assert_within_bf16_ulp(got, ref)


# ------------------------------------------------------------------------------------------------ attnpool_tokens
@pytest.mark.parametrize("n,HW,C", [(3, 49, 2048), (5, 1, 64), (9, 49, 200), (257, 4, 40)])
def test_attnpool_tokens(gpu_required, n, HW, C):
    """Row 0 = mean_s x_s + pos[0], row 1 + s = x_s + pos[1 + s], each within one bf16 ulp of fp64.  x has mean 4, so
    the mean token (~4, ulp 2^-5) is dominated by the mean: a divisor off by one (HW + 1 for HW = 49) moves it by 2.5
    ulps."""
    from marqo_b200.engine import debug_attnpool_tokens
    g = torch.Generator().manual_seed(n + HW + C)
    x = bf16(4.0 + torch.randn(n, HW, C, generator=g))
    pos = torch.randn(HW + 1, C, generator=g)
    got = torch.from_numpy(debug_attnpool_tokens(x.numpy(), pos.numpy()))
    xd, pd = x.double(), pos.double()
    ref = torch.cat([xd.mean(1, keepdim=True) + pd[0], xd + pd[1:]], dim=1)
    _assert_within_bf16_ulp(got, ref)


# ------------------------------------------------------------------------------------------------ im2col_f32
@pytest.mark.parametrize("n,S,p,cls", [(3, 224, 14, 1), (1, 224, 16, 0), (5, 224, 32, 1), (2, 256, 16, 0),
                                       (9, 224, 16, 1), (2, 224, 32, 0),
                                       # the ConvNeXt stems (patch 4, kpad 64), the served sizes above 256
                                       (2, 224, 4, 0), (2, 256, 4, 0), (1, 320, 4, 0), (1, 336, 14, 1), (1, 378, 14, 1),
                                       (1, 384, 16, 0), (1, 512, 16, 0)])
def test_im2col_f32(gpu_required, n, S, p, cls):
    """The ViT patch rows of fp32 CHW input, bit for bit the bf16 of the patch in k = c*p*p + dy*p + dx order (the
    order of conv1.weight.reshape(w, -1)); the class row (cls = 1) and the columns 3 p^2 .. kpad are zero."""
    from marqo_b200.engine import debug_im2col_f32
    g = torch.Generator().manual_seed(n + S + p + cls)
    K = 3 * p * p
    kpad = (K + 63) // 64 * 64   # the model's padding of conv1's K
    chw = torch.randn(n, 3, S, S, generator=g)
    got = torch.from_numpy(debug_im2col_f32(chw.numpy(), p, kpad, cls))
    patches = F.unfold(chw, kernel_size=p, stride=p).transpose(1, 2)   # [n, g*g, K], k = c*p*p + dy*p + dx
    rows = F.pad(patches, (0, kpad - K, cls, 0))                       # zero columns, then zero class rows on top
    assert torch.equal(got, bf16(rows.reshape(-1, kpad)))
