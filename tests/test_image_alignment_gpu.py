"""An image batch already on the device gives the same embeddings wherever it starts: the patch embedding reads the
uint8 pixels byte by byte, so a buffer that is not 16-byte aligned takes the same path as an aligned one."""
import numpy as np
import pytest
import torch

from oracle import encoders as E

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("patch", [32, 14])
def test_encode_images_u8_device_unaligned_is_bitwise_aligned(gpu_required, patch):
    from marqo_b200.engine import Encoder
    cfg = E.tiny_clip()
    cfg.vision.patch = patch
    sd = E.make_clip_weights(cfg, seed=21)
    tower = lambda t: dict(width=t.width, layers=t.layers, heads=t.heads, mlp=t.mlp, ctx=t.ctx, vocab=t.vocab,
                           image_size=t.image_size, patch=t.patch)
    enc = Encoder("clip", dict(embed_dim=cfg.embed_dim, act=cfg.act, mean=cfg.mean, std=cfg.std,
                               vision=tower(cfg.vision), text=tower(cfg.text)), sd, max_batch=4)
    n, S = 3, cfg.vision.image_size
    img = np.random.default_rng(patch).integers(0, 256, size=(n, S, S, 3), dtype=np.uint8)
    aligned = torch.from_numpy(img.reshape(-1)).cuda()
    shifted = torch.zeros(img.size + 16, dtype=torch.uint8, device="cuda")
    shifted[1:img.size + 1] = aligned                 # the same batch one byte past a 16-byte boundary
    assert aligned.data_ptr() % 16 == 0 and shifted.data_ptr() % 16 == 0
    out = torch.empty(2, n, cfg.embed_dim, dtype=torch.float32, device="cuda")
    enc.encode_images_u8_device(aligned.data_ptr(), n, S, S, out[0].data_ptr())
    enc.encode_images_u8_device(shifted.data_ptr() + 1, n, S, S, out[1].data_ptr())
    got = out.cpu()
    assert torch.isfinite(got).all()
    assert torch.equal(got[1], got[0])
    enc.close()
