"""GPU parity of the encoders (SURVEY §8 a2-a5) through the C ABI vs the CPU fp32 oracle (oracle/encoders.py) on the
same seeded weights and inputs.  Bar (BASELINE.json north_star): cosine >= 1 - 1e-3 per vector."""
import numpy as np
import pytest
import torch

import _checks as K
from oracle import encoders as E

pytestmark = pytest.mark.gpu


def _text_ids(g, n, ctx, vocab):
    ids = torch.zeros(n, ctx, dtype=torch.int64)
    for b in range(n):
        L = int(torch.randint(3, ctx + 1, (1,), generator=g))
        ids[b, 0] = vocab - 2
        ids[b, 1:L - 1] = torch.randint(1, vocab - 2, (L - 2,), generator=g)
        ids[b, L - 1] = vocab - 1
    return ids


@pytest.mark.parametrize("act", ["gelu", "quickgelu"])
def test_tiny_clip(gpu_required, act):
    from marqo_b200.engine import Encoder
    cfg = E.tiny_clip(act)
    sd = E.make_clip_weights(cfg, seed=11)
    enc = Encoder("clip", E.engine_config(cfg), sd, max_batch=8)
    g = torch.Generator().manual_seed(0)
    rng = np.random.default_rng(0)
    img = rng.integers(0, 256, size=(5, 224, 224, 3), dtype=np.uint8)
    px = E.clip_preprocess_u8(img)
    K.assert_embeddings_match(enc.encode_images_u8(img), E.clip_encode_image(sd, cfg, px))
    K.assert_embeddings_match(enc.encode_images_f32(px), E.clip_encode_image(sd, cfg, px))
    un = torch.from_numpy(enc.encode_images_u8(img, normalize=False))
    ref_un = E.clip_encode_image(sd, cfg, px, normalize=False)
    K.assert_embeddings_match(un, ref_un, unit_norm=False)
    assert torch.allclose(un.norm(dim=-1), ref_un.norm(dim=-1), rtol=2e-2)
    ids = _text_ids(g, 11, cfg.text.ctx, cfg.text.vocab)            # 11 > max_batch: exercises sub-batching
    K.assert_embeddings_match(enc.encode_tokens(ids.numpy()), E.clip_encode_text(sd, cfg, ids))
    # non-square input goes through the resize kernel; oracle goes through PIL
    big = rng.integers(0, 256, size=(2, 300, 400, 3), dtype=np.uint8)
    K.assert_embeddings_match(enc.encode_images_u8(big), E.clip_encode_image(sd, cfg, E.clip_preprocess_u8(big)))


@pytest.mark.parametrize("pool", ["mean", "cls"])
def test_tiny_bert(gpu_required, pool):
    from marqo_b200.engine import Encoder
    cfg = E.tiny_bert(pool)
    sd = E.make_bert_weights(cfg, seed=12)
    enc = Encoder("bert", E.engine_config(cfg), sd, max_batch=16)
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(1, cfg.vocab, (6, 40), generator=g)
    mask = torch.ones(6, 40, dtype=torch.int64)
    for b, L in enumerate([40, 3, 17, 1, 33, 40]):
        mask[b, L:] = 0
        ids[b, L:] = 0
    K.assert_embeddings_match(enc.encode_tokens(ids.numpy(), mask.numpy()), E.bert_encode(sd, cfg, ids, mask))
    K.assert_embeddings_match(enc.encode_tokens(ids.numpy()), E.bert_encode(sd, cfg, ids, None))


def test_repeated_small_calls_replay_cuda_graphs(gpu_required):
    """Small calls of one shape: 1st eager, 2nd captured into a CUDA graph, later ones replayed — with NEW inputs each
    time (the graph must read the staging buffers, not bake values in), interleaved with other shapes and towers."""
    from marqo_b200.engine import Encoder
    cfg = E.tiny_clip("gelu")
    sd = E.make_clip_weights(cfg, seed=13)
    enc = Encoder("clip", E.engine_config(cfg), sd, max_batch=8)
    g = torch.Generator().manual_seed(5)
    rng = np.random.default_rng(5)
    launches = []
    for it in range(5):
        ids = _text_ids(g, 3, cfg.text.ctx, cfg.text.vocab)
        K.assert_embeddings_match(enc.encode_tokens(ids.numpy()), E.clip_encode_text(sd, cfg, ids))
        launches.append(enc.last_timing()[1])
        img = rng.integers(0, 256, size=(2, 224, 224, 3), dtype=np.uint8)
        K.assert_embeddings_match(enc.encode_images_u8(img), E.clip_encode_image(sd, cfg, E.clip_preprocess_u8(img)))
        if it == 2:   # another shape in between does not disturb the cached graphs
            ids1 = _text_ids(g, 1, cfg.text.ctx, cfg.text.vocab)
            K.assert_embeddings_match(enc.encode_tokens(ids1.numpy()), E.clip_encode_text(sd, cfg, ids1))
        K.assert_embeddings_match(enc.encode_tokens(ids.numpy(), normalize=False),
                                  E.clip_encode_text(sd, cfg, ids, normalize=False), unit_norm=False)
    assert len(set(launches)) == 1          # the kernel count reported for a replayed graph is the eager one
    bcfg = E.tiny_bert("mean")
    bsd = E.make_bert_weights(bcfg, seed=14)
    benc = Encoder("bert", E.engine_config(bcfg), bsd, max_batch=16)
    for it in range(4):
        ids = torch.randint(1, bcfg.vocab, (4, 24), generator=g)
        mask = torch.ones(4, 24, dtype=torch.int64)
        L = int(torch.randint(1, 25, (1,), generator=g))
        mask[1, L:] = 0                       # the key-length mask changes between replays
        K.assert_embeddings_match(benc.encode_tokens(ids.numpy(), mask.numpy()), E.bert_encode(bsd, bcfg, ids, mask))


def test_vit_b_32(gpu_required):
    """BASELINE.json configs[1] architecture (open_clip/ViT-B-32), seeded weights, batch 8."""
    from marqo_b200.engine import Encoder
    cfg = E.CLIP_VIT_B_32
    sd = E.make_clip_weights(cfg, seed=1234)
    enc = Encoder("clip", E.engine_config(cfg), sd, max_batch=8)
    rng = np.random.default_rng(0)
    img = rng.integers(0, 256, size=(8, 224, 224, 3), dtype=np.uint8)
    K.assert_embeddings_match(enc.encode_images_u8(img), E.clip_encode_image(sd, cfg, E.clip_preprocess_u8(img)))
    ids = _text_ids(torch.Generator().manual_seed(2), 8, 77, cfg.text.vocab)
    K.assert_embeddings_match(enc.encode_tokens(ids.numpy()), E.clip_encode_text(sd, cfg, ids))


def test_e5_base_cfg1(gpu_required):
    """BASELINE.json configs[0]: hf/e5-base-v2 architecture, batch 8, 128 tokens (+ a ragged variant)."""
    from marqo_b200.engine import Encoder
    cfg = E.E5_BASE
    sd = E.make_bert_weights(cfg, seed=1234)
    enc = Encoder("bert", E.engine_config(cfg), sd, max_batch=8)
    g = torch.Generator().manual_seed(0)
    ids = torch.cat([torch.full((8, 1), 101), torch.randint(1000, 30000, (8, 126), generator=g), torch.full((8, 1), 102)], 1)
    K.assert_embeddings_match(enc.encode_tokens(ids.numpy()), E.bert_encode(sd, cfg, ids))
    mask = torch.ones(8, 128, dtype=torch.int64)
    for b, L in enumerate([16, 32, 48, 64, 80, 96, 112, 128]):
        mask[b, L:] = 0
        ids[b, L:] = 0
    K.assert_embeddings_match(enc.encode_tokens(ids.numpy(), mask.numpy()), E.bert_encode(sd, cfg, ids, mask))


def test_missing_weight_is_an_error(gpu_required):
    from marqo_b200._native import ERR_MISSING_WEIGHT
    cfg = E.tiny_bert()
    sd = E.make_bert_weights(cfg, seed=1)
    del sd["encoder.layer.1.output.dense.bias"]
    K.assert_refused("bert", E.engine_config(cfg), sd, ERR_MISSING_WEIGHT)


# ------------------------------------------------------------------------------------------------------------------
# Headline configurations (VERDICT r01 "weak #1"): parity measured on the shapes the performance numbers are quoted on.
# The GPU runs the full batch; the CPU oracle (fp32) restates a sample of it — positions spread over the batch, so a
# tile / sub-batch / persistent-scheduler bug anywhere in the batch shows up.
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cpu_threads():
    import os
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:                                   # cgroup v2 CPU quota: more threads than that only thrash
        quota, period = open("/sys/fs/cgroup/cpu.max").read().split()[:2]
        if quota != "max":
            n = min(n, max(1, -(-int(quota) // int(period))))
    except (OSError, ValueError):
        pass
    torch.set_num_threads(max(1, n))
    return n


def test_vit_l_14_image_batch_256(gpu_required, cpu_threads):
    """BASELINE.json metric / configs[2] shape: open_clip/ViT-L-14, 256 images per call, 224x224 uint8."""
    from marqo_b200.engine import Encoder
    cfg = E.CLIP_VIT_L_14
    sd = E.make_clip_weights(cfg, seed=1234)
    vis = {k: v for k, v in sd.items() if k.startswith("visual.")}
    enc = Encoder("clip", dict(E.engine_config(cfg), text=None), vis, max_batch=256)
    rng = np.random.default_rng(0)
    img = rng.integers(0, 256, size=(256, 224, 224, 3), dtype=np.uint8)
    got = enc.encode_images_u8(img)
    assert got.shape == (256, 768) and np.isfinite(got).all()
    np.testing.assert_allclose(np.linalg.norm(got, axis=1), 1.0, atol=1e-5)
    pos = K.sample_positions(256, 3)
    ref = E.clip_encode_image(sd, cfg, E.clip_preprocess_u8(img[pos]))
    K.assert_embeddings_match(got[pos], ref)
    # the same images in a different batch composition give the same vectors (no cross-item leakage)
    again = enc.encode_images_u8(img[pos])
    assert float((1 - K.cosine(again, got[pos])).max()) < 1e-5
    enc.close()


def test_vit_l_14_text_batch_64(gpu_required, cpu_threads):
    """The caption half of configs[2]: ViT-L-14 text tower (width 768, 12 layers, S = 77, causal, EOT pooling)."""
    from marqo_b200.engine import Encoder
    cfg = E.CLIP_VIT_L_14
    sd = E.make_clip_weights(cfg, seed=1234)
    txt = {k: v for k, v in sd.items() if not k.startswith("visual.")}
    enc = Encoder("clip", dict(E.engine_config(cfg), vision=None), txt, max_batch=64)
    ids = _text_ids(torch.Generator().manual_seed(3), 64, 77, cfg.text.vocab)
    ids[5, :] = 0
    ids[5, 0], ids[5, 1] = cfg.text.vocab - 2, cfg.text.vocab - 1           # shortest possible text
    got = enc.encode_tokens(ids.numpy())
    pos = K.sample_positions(64, 3) + [5]
    K.assert_embeddings_match(got[pos], E.clip_encode_text(sd, cfg, ids[pos]))
    enc.close()


def test_vit_b_32_batch_256_image_and_text(gpu_required, cpu_threads):
    """BASELINE.json configs[1]: open_clip/ViT-B-32 image + text vectorise at batch 256 (S = 50 / 77: the
    short-sequence attention path)."""
    from marqo_b200.engine import Encoder
    cfg = E.CLIP_VIT_B_32
    sd = E.make_clip_weights(cfg, seed=1234)
    enc = Encoder("clip", E.engine_config(cfg), sd, max_batch=256)
    rng = np.random.default_rng(1)
    img = rng.integers(0, 256, size=(256, 224, 224, 3), dtype=np.uint8)
    got = enc.encode_images_u8(img)
    pos = K.sample_positions(256, 4)
    K.assert_embeddings_match(got[pos], E.clip_encode_image(sd, cfg, E.clip_preprocess_u8(img[pos])))
    ids = _text_ids(torch.Generator().manual_seed(4), 256, 77, cfg.text.vocab)
    gt = enc.encode_tokens(ids.numpy())
    K.assert_embeddings_match(gt[pos], E.clip_encode_text(sd, cfg, ids[pos]))
    big = rng.integers(0, 256, size=(16, 480, 640, 3), dtype=np.uint8)        # SURVEY §8(d): exercises bicubic + crop
    gb = enc.encode_images_u8(big)
    K.assert_embeddings_match(gb[[0, 15]], E.clip_encode_image(sd, cfg, E.clip_preprocess_u8(big[[0, 15]])))
    enc.close()


def test_e5_large_512_tokens(gpu_required, cpu_threads):
    """BASELINE.json configs[3]: hf/e5-large-v2 architecture, 512-token chunks — full length and 50 % padded."""
    from marqo_b200.engine import Encoder
    cfg = E.E5_LARGE
    sd = E.make_bert_weights(cfg, seed=1234)
    enc = Encoder("bert", E.engine_config(cfg), sd, max_batch=8)
    g = torch.Generator().manual_seed(0)
    ids = torch.cat([torch.full((8, 1), 101), torch.randint(1000, 30000, (8, 510), generator=g), torch.full((8, 1), 102)], 1)
    got = enc.encode_tokens(ids.numpy())
    K.assert_embeddings_match(got[[7]], E.bert_encode(sd, cfg, ids[[7]]))
    mask = torch.ones(8, 512, dtype=torch.int64)
    for b, L in enumerate([256, 200, 312, 256, 1, 511, 256, 300]):           # ~50 % padding, ragged
        mask[b, L:] = 0
        ids[b, L:] = 0
    gm = enc.encode_tokens(ids.numpy(), mask.numpy())
    sel = [4, 5]
    K.assert_embeddings_match(gm[sel], E.bert_encode(sd, cfg, ids[sel], mask[sel]))
    enc.close()
