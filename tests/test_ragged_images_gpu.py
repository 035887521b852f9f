"""Images of mixed sizes in one call, on the GPU: the ragged resize against Pillow bit for bit at every served S in
both modes; every vision kind's ragged entry points (host, and device at sync 1 and 0) against the uniform entry point
on the Pillow-resized stack, bit for bit; sub-batching; launch counts; refusals; and encode_to_device /
add_documents_device over mixed sizes."""
import ctypes as C
import io

import numpy as np
import pytest
import torch

import _coca_oracle as CO
from _checks import served_resize_sizes
from marqo_b200 import _native as N

pytestmark = pytest.mark.gpu

# identity, smaller than S on one axis and on both (upscale), portrait and landscape downscales, odd sizes, the
# one-pixel strips and a 12 MP photo
def _mixed_sizes(S):
    return [(S, S), (S // 2, S + 77), (S // 3, S // 2 + 1), (640, 480), (480, 640), (333, 517), (S + 1, S - 1),
            (1, 997), (997, 1), (3000, 4000)]


def _pillow(a, S, squash):
    """uint8 [h, w, 3] -> [S, S, 3] as the reference preprocessing resizes: torchvision Resize(S, BICUBIC) +
    CenterCrop(S) on a PIL image, or the squash as one call of Pillow's two-pass resampler (PIL resize((S, S),
    BICUBIC) for an image of ordinary shape; see test_siglip_gpu for the very tall ones)."""
    from PIL import Image
    from torchvision.transforms import CenterCrop, InterpolationMode, Resize
    im = Image.fromarray(a)
    if squash:
        return np.asarray(im._new(im.im.resize((S, S), Image.BICUBIC, (0, 0) + im.size)))
    for t in (Resize(S, interpolation=InterpolationMode.BICUBIC), CenterCrop(S)):
        im = t(im)
    return np.asarray(im.convert("RGB"))


def _images(sizes, seed):
    rng = np.random.default_rng(seed)
    out = []
    for i, (h, w) in enumerate(sizes):
        if i % 2:   # smooth gradients beside the noise
            a = (np.linspace(0, 255, w)[None, :, None] * np.ones((h, 1, 3))).astype(np.uint8)
            a[..., 1] = (np.linspace(255, 0, h)[:, None] * np.ones((1, w))).astype(np.uint8)
        else:
            a = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        out.append(a)
    return out


@pytest.mark.parametrize("mode", ["crop", "squash"])
def test_ragged_resize_matches_pillow_bit_exact(gpu_required, mode):
    from marqo_b200.engine import debug_resize_ragged
    for S in served_resize_sizes(mode):
        imgs = _images(_mixed_sizes(S), S)
        got = debug_resize_ragged(imgs, S, squash=mode == "squash")
        for a, g in zip(imgs, got):
            np.testing.assert_array_equal(g, _pillow(a, S, mode == "squash"), err_msg=f"S = {S}, {a.shape}")


# (kind, registry name, arch edits): one seeded model of every vision kind that takes uint8 images, one layer deep
_KINDS = {
    "clip": ("clip", "open_clip/ViT-B-32/laion2b_s34b_b79k", {"vision.layers": 1, "text": None}),
    "big_vit_squash": ("clip", "open_clip/ViT-H-14-quickgelu/dfn5b", {"vision.layers": 1, "text": None}),
    "siglip": ("siglip", "open_clip/ViT-B-16-SigLIP/webli", {"vision.layers": 1, "text": None}),
    "eva02": ("clip_eva", "open_clip/EVA02-B-16/merged2b_s8b_b131k", {"layers": 0, "eva.layers": 1}),
    "coca": ("clip", CO.B32, {"vision.layers": 1, "text": None}),
    "resnet": ("clip_resnet", "open_clip/RN50/openai", {"layers": 0, "resnet.layers": [1, 1, 1, 1]}),
    "convnext": ("clip_convnext", "open_clip/convnext_base_w/laion2b_s13b_b82k",
                 {"layers": 0, "convnext.depths": [1, 1, 1, 1]}),
}


def _encoder(name, max_batch=16):
    from marqo_b200 import model_registry as R
    from marqo_b200.engine import Encoder
    from marqo_b200.weights import random_weights
    kind, model, edits = _KINDS[name]
    arch = R.get_model_properties(model)["arch"]
    for path, value in edits.items():
        *outer, key = path.split(".")
        d = arch
        for k in outer:
            d = d[k]
        d[key] = value
    squash = kind == "siglip" or arch.get("resize_mode") == "squash"
    return Encoder(kind, arch, random_weights(kind, arch, 11), max_batch=max_batch), squash


def _uniform_of_pillow(enc, imgs, squash, normalize=True):
    """encode_images_u8 of the Pillow-resized stack: what the ragged calls must return bit for bit."""
    S = enc.image_size
    return enc.encode_images_u8(np.stack([_pillow(a, S, squash) for a in imgs]), normalize)


def _jpegs(sizes, seed):
    from PIL import Image
    out = []
    for a in _images(sizes, seed):
        buf = io.BytesIO()
        Image.fromarray(a).save(buf, format="JPEG", quality=90)
        out.append(buf.getvalue())
    return out


def _ragged_device(enc, tensors, sync, normalize=True):
    out = torch.full((len(tensors), enc.embed_dim), float("nan"), device="cuda")
    torch.cuda.synchronize()
    enc.encode_images_u8_ragged_device([t.data_ptr() for t in tensors], [t.shape[0] for t in tensors],
                                       [t.shape[1] for t in tensors], out.data_ptr(), normalize=normalize,
                                       sync=sync)
    if not sync:
        torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("name", list(_KINDS))
def test_ragged_towers_match_the_uniform_call_bit_exact(gpu_required, name):
    from marqo_b200.image_decode import decode_images_to_device
    enc, squash = _encoder(name)
    try:
        S = enc.image_size
        imgs = _images([(S, S), (480, 640), (640, 480), (S // 2, S // 3), (333, 517), (S + 1, S - 1), (1, 997),
                        (997, 1), (480, 640)], 5)
        for normalize in (True, False):
            got = enc.encode_images_u8_ragged(imgs, normalize)
            assert got.shape == (len(imgs), enc.embed_dim) and np.isfinite(got).all()
            np.testing.assert_array_equal(got, _uniform_of_pillow(enc, imgs, squash, normalize))
        # device-resident pixels, as the GPU JPEG decoder leaves them
        dev = decode_images_to_device(_jpegs([(240, 320), (320, 240), (S, S), (181, 263), (64, 96)], 6), device=0)
        want = _uniform_of_pillow(enc, [t.cpu().numpy() for t in dev], squash)
        for sync in (True, False):
            np.testing.assert_array_equal(_ragged_device(enc, dev, sync), want)
    finally:
        enc.close()


def test_sub_batches_land_in_order(gpu_required):
    """max_batch 4 and 11 images of mixed sizes: three sub-batches, each row the uniform call's."""
    enc, squash = _encoder("clip", max_batch=4)
    try:
        S = enc.image_size
        imgs = _images([(480, 640), (S, S), (100, 150), (640, 480), (333, 517), (S + 9, S), (77, 500), (500, 77),
                        (S, S + 3), (300, 300), (1000, 750)], 7)
        want = _uniform_of_pillow(enc, imgs, squash)
        assert len(np.unique(want, axis=0)) == len(imgs)
        np.testing.assert_array_equal(enc.encode_images_u8_ragged(imgs), want)
        dev = [torch.from_numpy(a).cuda() for a in imgs]
        np.testing.assert_array_equal(_ragged_device(enc, dev, True), want)
    finally:
        enc.close()


def test_launches_do_not_depend_on_the_sizes(gpu_required):
    """A ragged call launches what a uniform call of the same n on images of another size than S does (the resize's
    two kernels, then the tower), whether its images have one size or 16."""
    enc, _ = _encoder("clip")
    try:
        S, n = enc.image_size, 16
        rng = np.random.default_rng(8)
        enc.encode_images_u8(rng.integers(0, 256, (n, S + 37, S - 21, 3), dtype=np.uint8))
        uniform = enc.last_timing()[1]
        enc.encode_images_u8_ragged(_images([(S + 37, S - 21)] * n, 8))
        one = enc.last_timing()[1]
        enc.encode_images_u8_ragged(_images([(S - 50 + 13 * i, S + 40 - 7 * i) for i in range(n)], 9))
        sixteen = enc.last_timing()[1]
        assert uniform == one == sixteen > 2
    finally:
        enc.close()


def test_refusals_write_nothing(gpu_required):
    from marqo_b200.engine import Encoder
    from oracle import encoders as E
    enc, _ = _encoder("clip")
    lib = N.load()
    h = enc._handle()
    img = np.zeros((40, 50, 3), np.uint8)
    d_img = torch.zeros((40, 50, 3), dtype=torch.uint8, device="cuda")
    out = np.full((2, enc.embed_dim), np.nan, np.float32)
    d_out = torch.full((2, enc.embed_dim), float("nan"), device="cuda")
    torch.cuda.synchronize()

    def arrays(ptr, hs=(40, 40), ws=(50, 50)):
        return ((C.c_void_p * 2)(ptr, ptr), np.array(hs, np.int32), np.array(ws, np.int32))

    def host(m, p, hs, ws, n):
        return lib.b200_model_encode_images_u8_ragged(m, p, None if hs is None else hs.ctypes.data_as(C.c_void_p),
                                                      None if ws is None else ws.ctypes.data_as(C.c_void_p), n, 1,
                                                      out.ctypes.data_as(C.c_void_p))

    def device(m, p, hs, ws, n):
        return lib.b200_model_encode_images_u8_ragged_device(
            m, p, None if hs is None else hs.ctypes.data_as(C.c_void_p),
            None if ws is None else ws.ctypes.data_as(C.c_void_p), n, 1, C.c_void_p(d_out.data_ptr()), 1)

    try:
        for call, ptr in ((host, img.ctypes.data), (device, d_img.data_ptr())):
            p, hs, ws = arrays(ptr)
            cases = {"NULL images": (None, hs, ws, 2), "NULL heights": (p, None, ws, 2), "NULL widths": (p, hs, None, 2),
                     "NULL entry": ((C.c_void_p * 2)(ptr, None), hs, ws, 2), "n = 0": (p, hs, ws, 0),
                     "n < 0": (p, hs, ws, -1), "height 0": arrays(ptr, hs=(40, 0)) + (2,),
                     "width < 0": arrays(ptr, ws=(-50, 50)) + (2,)}
            for what, args in cases.items():
                assert call(h, *args) == N.ERR_INVALID_ARG, (call.__name__, what)
        cfg = E.tiny_bert()
        bert = Encoder("bert", dict(width=cfg.width, layers=cfg.layers, heads=cfg.heads, mlp=cfg.mlp, vocab=cfg.vocab,
                                    max_pos=cfg.max_pos, type_vocab=cfg.type_vocab, pool="mean"),
                       E.make_bert_weights(cfg, seed=4), max_batch=2)
        try:
            assert host(bert._handle(), *arrays(img.ctypes.data), 2) == N.ERR_INVALID_ARG
            assert device(bert._handle(), *arrays(d_img.data_ptr()), 2) == N.ERR_INVALID_ARG
        finally:
            bert.close()
        assert np.isnan(out).all() and torch.isnan(d_out).all()
    finally:
        enc.close()


def _loader(enc):
    from marqo_b200.loaders import B200OpenCLIP
    loader = B200OpenCLIP.__new__(B200OpenCLIP)
    loader.model, loader.model_properties = enc, {"max_batch": 16}
    return loader


def test_fast_path_takes_mixed_sizes(gpu_required):
    """encode_to_device over mixed-size CUDA tensors and numpy arrays, and add_documents_device over a ragged
    device_contents list: the rows of the uniform call on the Pillow-resized stack, in input order."""
    from marqo_b200.add_documents import add_documents_device
    from marqo_b200.gpu_tensor_index import GpuTensorIndex
    from marqo_b200.image_decode import decode_images_to_device
    enc, squash = _encoder("clip")
    try:
        S = enc.image_size
        imgs = _images([(480, 640), (S, S), (100, 150), (640, 480), (333, 517), (S + 9, S), (77, 500)], 10)
        want = _uniform_of_pillow(enc, imgs, squash)
        loader = _loader(enc)
        dev = [torch.from_numpy(a).cuda() for a in imgs]
        for items in (dev, imgs):
            got = loader.encode_to_device(items, default="image")
            assert got.is_cuda
            np.testing.assert_array_equal(got.cpu().numpy(), want)

        decoded = decode_images_to_device(_jpegs([(240, 320), (320, 240), (S, S), (181, 263)], 11), device=0)
        rows = _uniform_of_pillow(enc, [t.cpu().numpy() for t in decoded], squash)
        ix = GpuTensorIndex()
        try:
            docs = [{"_id": f"d{i}", "img": f"http://example.com/{i}.jpg"} for i in range(len(decoded))]
            r = add_documents_device(ix, "s1", docs, {"img": (loader, "image")}, device_contents={"img": decoded})
            assert not r.errors
            got = ix.get_batch([d["_id"] for d in docs], "s1")
            for i, resp in enumerate(got.responses):
                v = np.asarray(resp.document.fields["marqo__embeddings_img"]["0"], np.float32)
                np.testing.assert_allclose(v, rows[i], rtol=0, atol=1e-3)   # the store keeps fp16
                assert int(np.argmax(rows @ v)) == i
        finally:
            ix.close()
    finally:
        enc.close()
