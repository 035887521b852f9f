"""OWL-ViT's detection kernels on the H100 against fp64, and the shared stages at the detector's shapes: the 240 -> 768
and 240 -> 840 squash against Pillow bit for bit, the gather patch embedding bit for bit at 768/32, 768/16 and 840/14,
and attention at 577, 2305 and 3601 tokens within the fp64 bound of test_attention_exact_gpu."""
import math

import numpy as np
import pytest
import torch

from _checks import bf16

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available(), reason="needs an H100 (sm_90a)")]


def _ln64(x, g, b, eps=1e-5):
    x = x.double()
    m = x.mean(-1, keepdim=True)
    v = ((x - m) ** 2).mean(-1, keepdim=True)
    return (x - m) / torch.sqrt(v + eps) * g.double() + b.double()


@pytest.mark.parametrize("n,G,w", [(2, 4, 768), (3, 24, 768), (1, 60, 1024)])
def test_merge_ln_against_fp64(gpu_required, n, G, w):
    """bf16 output of LN_det(LN_post(patch) * LN_post(class)) within one bf16 rounding of fp64 (plus fp32 slack)."""
    from marqo_b200.engine import debug_owl_merge_ln
    g = torch.Generator().manual_seed(G + w)
    N = G * G + 1
    x = torch.randn(n * N, w, generator=g) * 3 + torch.randn(w, generator=g)
    pg, pb, dg, db = (torch.randn(w, generator=g) * 0.3 + (1 if i % 2 == 0 else 0) for i in range(4))
    got = torch.from_numpy(debug_owl_merge_ln(x.numpy(), N, pg.numpy(), pb.numpy(), dg.numpy(), db.numpy()))
    e = _ln64(x, pg, pb).view(n, N, w)
    want = _ln64(e[:, 1:] * e[:, :1], dg, db).reshape(n * G * G, w)
    err = (got.double() - want).abs()
    bound = 2.0**-8 * want.abs() + 1e-4 * (1 + dg.double().abs())
    assert bool((err <= bound).all()), float((err / bound).max())


def _class_inputs(M, E, ldc, seed, scale_shift=0.0):
    g = torch.Generator().manual_seed(seed)
    c = torch.randn(M, ldc, generator=g)
    c[:, E + 1] = torch.randn(M, generator=g) * 3 + scale_shift   # logit_scale: both ELU branches
    t = torch.randn(E, generator=g) * 5
    return c, t


def _class64(c, t, E):
    c, t = c.double(), t.double()
    cc = c[:, :E]
    ch = cc / (cc.norm(dim=-1, keepdim=True) + 1e-6)
    u = t / t.norm()
    q = u / (u.norm() + 1e-6)
    s = c[:, E + 1]
    return ((ch @ q) + c[:, E]) * (torch.where(s > 0, s, torch.expm1(s)) + 1)


@pytest.mark.parametrize("M,E,ldc", [(577 - 1, 512, 576), (3600, 768, 832), (37, 512, 576)])
def test_class_logits_against_fp64(gpu_required, M, E, ldc):
    from marqo_b200.engine import debug_owl_class_logits
    c, t = _class_inputs(M, E, ldc, M + E)
    got = torch.from_numpy(debug_owl_class_logits(c.numpy(), E, t.numpy())).double()
    want = _class64(c, t, E)
    s = c[:, E + 1]
    assert bool((s > 0).any()) and bool((s < 0).any()), "both ELU branches"
    scale = torch.where(s > 0, s, torch.expm1(s)).double() + 1
    bound = 1e-5 * (1 + c[:, E].double().abs()) * scale + 1e-6
    assert bool(((got - want).abs() <= bound).all()), float(((got - want).abs() / bound).max())


def test_class_logits_zero_rows_use_the_epsilon(gpu_required):
    """A zero dense0 row has |c| = 0: c^ = 0 / (0 + 1e-6) = 0, not NaN, so the logit is shift * (ELU(scale) + 1), up
    to expm1f's last bit."""
    from marqo_b200.engine import debug_owl_class_logits
    E, ldc = 512, 576
    c, t = _class_inputs(16, E, ldc, 5)
    c[:, :E] = 0
    got = debug_owl_class_logits(c.numpy(), E, t.numpy())
    s = c[:, E + 1].numpy()
    want = c[:, E].numpy() * (np.where(s > 0, s, np.expm1(s)) + np.float32(1))
    np.testing.assert_allclose(got, want, rtol=5e-7, atol=0)


@pytest.mark.parametrize("M,w,P", [(576 * 2, 768, 576), (3600, 1024, 3600), (9, 768, 9)])
def test_boxes_against_fp64(gpu_required, M, w, P):
    from marqo_b200.engine import debug_owl_boxes, owl_box_bias
    g = torch.Generator().manual_seed(M + w)
    a = bf16(torch.randn(M, w, generator=g))
    w2 = torch.randn(4, w, generator=g) / math.sqrt(w)
    b2 = torch.randn(4, generator=g)
    G = int(math.isqrt(P))
    bb = torch.from_numpy(owl_box_bias(G))
    got = torch.from_numpy(debug_owl_boxes(a.numpy(), P, w2.numpy(), b2.numpy(), bb.numpy())).double()
    z = a.double() @ w2.double().t() + b2.double() + bb.double().repeat(M // P, 1)
    want = torch.sigmoid(z)
    assert bool(((got - want).abs() <= 1e-6 + 1e-6 * want).all()), float((got - want).abs().max())


def test_boxes_saturate(gpu_required):
    """Huge pre-activations give exactly 0 and 1, never NaN: expf(-z) overflows to inf for z << 0."""
    from marqo_b200.engine import debug_owl_boxes
    w, P = 128, 4
    a = torch.ones(P, w)
    w2 = torch.zeros(4, w)
    w2[0], w2[1] = 10.0, -10.0
    got = debug_owl_boxes(a.numpy(), P, w2.numpy(), np.zeros(4, np.float32), np.zeros((P, 4), np.float32))
    assert (got[:, 0] == 1.0).all() and (got[:, 1] == 0.0).all() and (got[:, 2:] == 0.5).all()


# --------------------------------------------------------------------------- the shared stages at OWL-ViT's shapes
@pytest.mark.parametrize("S", [768, 840])
def test_squash_240_matches_pillow(gpu_required, S):
    from test_ragged_images_gpu import _pillow
    from marqo_b200.engine import debug_resize_squash
    rng = np.random.default_rng(S)
    a = rng.integers(0, 256, (3, 240, 240, 3), dtype=np.uint8)
    got = debug_resize_squash(a, S)
    for i in range(3):
        np.testing.assert_array_equal(got[i], _pillow(a[i], S, True))


@pytest.mark.parametrize("S,p,N", [(768, 32, 768), (768, 16, 768), (840, 14, 1024)])
def test_patch_embed_bit_exact(gpu_required, S, p, N):
    import test_patch_embed_gpu as PE
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    PE.test_gather_is_exact(gpu_required, sms, S, p, N, PE.CLS, *PE.OPENAI, 1)


@pytest.mark.parametrize("S,Hn,B", [(577, 12, 2), (2305, 12, 1), (3601, 16, 1)])
def test_attention_within_bound(gpu_required, S, Hn, B):
    import test_attention_exact_gpu as A
    hd = 64
    W = Hn * hd
    x = A._family_inputs("peaked", B, S, Hn, hd, seed=S)
    got = A._attention(x.reshape(B * S, 3 * W).to(torch.bfloat16), B, S, Hn, A.NONE)
    got = got.view(B, S, Hn, hd).permute(0, 2, 1, 3).double()
    q, k, v = x.permute(2, 0, 3, 1, 4)
    keep = torch.ones(B, 1, S, S, dtype=torch.bool, device="cuda")
    c = math.log2(math.e) / math.sqrt(hd)
    ratio = A._within_bound(got, q, k, v, keep, None, hd, c, A._nkb(S, A.NONE, [S] * B), S, True)
    print(f"\n[owl attention bound] S={S} H={Hn}: worst ratio {ratio:.4f}")
