"""encode_to_device's routing of image sub-batches, with a fake encoder standing in for the native one: a sub-batch of
mixed sizes makes one ragged call with every image's pointer and size in input order, and a sub-batch of one size
still makes one encode_images_u8_device call over its stacked block.  Host tensors stand in for device ones, so the
'device' pointers are readable through ctypes."""
import ctypes

import numpy as np
import torch

from marqo_b200.loaders import B200OpenCLIP

E = 4


def _pixels(ptr, h, w):
    return np.ctypeslib.as_array((ctypes.c_uint8 * (h * w * 3)).from_address(ptr)).reshape(h, w, 3).copy()


def _rows(ptr, n):
    return np.ctypeslib.as_array((ctypes.c_float * (n * E)).from_address(ptr)).reshape(n, E)


class FakeEncoder:
    """Records each call; row i of a call's output = (sum of image i's pixels, h, w, normalize)."""
    device, embed_dim, image_size = 0, E, 224

    def __init__(self):
        self.calls = []

    def encode_images_u8_device(self, d_ptr, n, h, w, d_out_ptr, normalize=True, sync=True):
        imgs = [_pixels(d_ptr + i * h * w * 3, h, w) for i in range(n)]
        self.calls.append(("uniform", imgs, sync))
        _rows(d_out_ptr, n)[:] = [[int(a.sum()), h, w, float(normalize)] for a in imgs]

    def encode_images_u8_ragged_device(self, ptrs, heights, widths, d_out_ptr, normalize=True, sync=True):
        imgs = [_pixels(p, h, w) for p, h, w in zip(ptrs, heights, widths)]
        self.calls.append(("ragged", imgs, sync))
        _rows(d_out_ptr, len(ptrs))[:] = [[int(a.sum()), a.shape[0], a.shape[1], float(normalize)] for a in imgs]


def _loader(monkeypatch, on_device):
    loader = B200OpenCLIP.__new__(B200OpenCLIP)
    loader.model = FakeEncoder()
    loader.model_properties = {}
    monkeypatch.setattr(B200OpenCLIP, "_on_model_device", lambda self, it: on_device and isinstance(it, torch.Tensor))
    monkeypatch.setattr(B200OpenCLIP, "_sync_device", staticmethod(lambda device: None))
    monkeypatch.setattr(B200OpenCLIP, "_torch_device", lambda self: torch.device("cpu"))
    return loader


def _images(sizes, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, generator=g) for h, w in sizes]


def _check(out, calls, imgs, normalize):
    """Every row of out belongs to its own image, and the calls saw the images in input order."""
    assert out.shape == (len(imgs), E)
    for i, t in enumerate(imgs):
        assert out[i].tolist() == [float(t.sum()), t.shape[0], t.shape[1], float(normalize)]
    seen = [a for _, batch, _ in calls for a in batch]
    assert len(seen) == len(imgs) and all(np.array_equal(a, t.numpy()) for a, t in zip(seen, imgs))
    assert all(sync for _, _, sync in calls)


def test_mixed_sizes_make_one_ragged_call_per_sub_batch(monkeypatch):
    sizes = [(8, 8), (6, 10), (8, 8), (5, 3), (1, 9), (9, 1), (8, 8), (7, 7), (6, 10), (2, 2), (3, 4)]
    imgs = _images(sizes, 0)
    for on_device in (True, False):   # CUDA tensors by pointer, or host arrays through one packed upload
        loader = _loader(monkeypatch, on_device)
        items = imgs if on_device else [t.numpy() for t in imgs]
        out = loader.encode_to_device(items, default="image", normalize=False, sub_batch=4)
        calls = loader.model.calls
        assert [k for k, _, _ in calls] == ["ragged"] * 3
        assert [len(b) for _, b, _ in calls] == [4, 4, 3]
        _check(out, calls, imgs, False)


def test_host_images_are_packed_back_to_back(monkeypatch):
    """The host arrays of a mixed sub-batch reach the ragged call as one upload: consecutive pointers step by the
    previous image's bytes."""
    loader = _loader(monkeypatch, False)
    sizes = [(4, 6), (3, 3), (5, 2)]
    seen = []
    real = FakeEncoder.encode_images_u8_ragged_device

    def spy(self, ptrs, heights, widths, *a, **kw):
        seen.append((list(ptrs), list(heights), list(widths)))
        return real(self, ptrs, heights, widths, *a, **kw)

    monkeypatch.setattr(FakeEncoder, "encode_images_u8_ragged_device", spy)
    imgs = _images(sizes, 1)
    out = loader.encode_to_device([t.numpy() for t in imgs], default="image")
    (ptrs, heights, widths), = seen
    assert heights == [4, 3, 5] and widths == [6, 3, 2]
    assert [b - a for a, b in zip(ptrs, ptrs[1:])] == [4 * 6 * 3, 3 * 3 * 3]
    _check(out, loader.model.calls, imgs, True)


def test_single_size_sub_batches_keep_the_uniform_call(monkeypatch):
    """A sub-batch of one size keeps encode_images_u8_device, also when the next sub-batch mixes sizes."""
    sizes = [(8, 8)] * 4 + [(8, 8), (6, 10), (8, 8), (6, 10)] + [(6, 10)] * 2
    imgs = _images(sizes, 2)
    for on_device in (True, False):
        loader = _loader(monkeypatch, on_device)
        items = imgs if on_device else [t.numpy() for t in imgs]
        out = loader.encode_to_device(items, default="image", sub_batch=4)
        calls = loader.model.calls
        assert [(k, len(b)) for k, b, _ in calls] == [("uniform", 4), ("ragged", 4), ("uniform", 2)]
        _check(out, calls, imgs, True)
