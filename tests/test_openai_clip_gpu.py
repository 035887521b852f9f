"""The OpenAI CLIP models of the `clip` and `fp16_clip` loaders on the GPU:

  - the GEMM's K and N tails (K % 8, bf16 N % 8) through the 1 x 1 conv path, against fp64 and bit for bit against
    the same GEMM on explicitly zero-padded operands at K = 64 ceil(K / 64);
  - every distinct convolution of RN50x4, RN50x16 and RN50x64 (the 3 x 3 gather at cin 40 ... 768) against fp64, and
    the gather's border halo at cin 40 and 48;
  - the RN50x16, RN50x64 and RN50x4 towers and ViT-L/14@336px through the C ABI against the fp32 oracles on every
    input path, and their text towers;
  - vectorise of each `clip` name against its open_clip twin on the same weights (bit for bit), `fp16/*` as the fp32
    name's vectors rounded to float16, and a custom RN50x16 checkpoint through vectorise -> GpuTensorIndex against
    the score oracle, and the resize at the wide ResNets' sizes against Pillow;
  - with MARQO_B200_BASELINE_LIB naming a library built from an earlier commit, RN50's output on a seeded batch
    against that library's, bit for bit.

The full-size oracles run on the GPU in fp32 with TF32 off, on a few rows of each batch (rows are independent)."""
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import _big_vit_oracle as BV
import _checks as K
import _resnet_oracle as O
from _checks import fp32_oracle  # noqa: F401 (autouse)
from oracle import encoders as E

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]


def _arch(name):
    from marqo_b200 import model_registry as R
    return R.WIDE_RESNET_ARCHS[name] if name in R.WIDE_RESNET_ARCHS else R.get_model_properties(name)["arch"]


def _wide_weights(a, seed):
    """Seeded random weights of a wide ResNet with every bottleneck's residual branch (bn3) scaled by 1 / 4, as
    trained ResNets keep theirs small.  With unit-gain random branches the 40 to 64 blocks grow one component common
    to every image: the oracle's embeddings of different images then agree to 3e-3 and the cosine to the oracle
    measures the bf16 rounding of that sum rather than the kernels; that is depth, not width: RN50x16's blocks at
    width 64, which run only the power-of-two paths, err by up to 7e-4 too, and at RN50's depth width 96 errs by
    1e-5 as width 64 does."""
    from marqo_b200.weights import random_clip_resnet_weights
    sd = random_clip_resnet_weights(a, seed=seed)
    for k in sd:
        if ".bn3." in k and k.rsplit(".", 1)[1] in ("weight", "bias"):
            sd[k] = sd[k] * np.float32(0.25)
    return sd


# ------------------------------------------------------------------------------------------------------------------
# GEMM K and N tails: a 1 x 1 conv is the plain GEMM over the NHWC pixel rows (K = cin, N = cout, bf16 output)
# ------------------------------------------------------------------------------------------------------------------
def _pad_channels(a, axis, to):
    pad = [(0, 0)] * a.ndim
    pad[axis] = (0, to - a.shape[axis])
    return np.pad(a, pad)


@pytest.mark.parametrize("N", [8, 40, 48, 80])
@pytest.mark.parametrize("Kd", [8, 40, 80, 96, 200])
def test_gemm_k_and_n_tails(gpu_required, Kd, N):
    from marqo_b200.engine import debug_conv2d
    g = torch.Generator().manual_seed(Kd * 100 + N)
    n, H = 2, 9   # M = 162: a full and a partial row tile, straddling the images
    x = torch.relu(torch.randn(n, H, H, Kd, generator=g)).numpy()
    w = (torch.randn(N, Kd, 1, 1, generator=g) / Kd ** 0.5).numpy()
    b = (torch.randn(N, generator=g) * 0.1).numpy()
    res = torch.randn(n, H, H, N, generator=g).numpy()
    Kp = -(-Kd // 64) * 64
    xp, wp = _pad_channels(x, 3, Kp), _pad_channels(w, 1, Kp)
    prod = K.bf16(torch.from_numpy(x)).double() @ K.bf16(torch.from_numpy(w)).double().reshape(N, Kd).T + \
        torch.from_numpy(b).double()
    scale = float(prod.abs().max())
    for relu, r in ((False, None), (True, None), (True, res)):
        got = debug_conv2d(x, w, b, r, relu=relu)
        padded = debug_conv2d(xp, wp, b, r, relu=relu)
        np.testing.assert_array_equal(got, padded)
        ref = prod + (K.bf16(torch.from_numpy(r)).double() if r is not None else 0)
        if relu:
            ref = torch.relu(ref)
        assert np.isfinite(got).all()
        torch.testing.assert_close(torch.from_numpy(got).double(), ref, rtol=2 ** -7, atol=1e-3 * scale)


# ------------------------------------------------------------------------------------------------------------------
# Every distinct convolution of the wide ResNets: (cin, cout, k, H), the strided blocks' 3 x 3 before their pool
# ------------------------------------------------------------------------------------------------------------------
def _conv_shapes(width, S):
    w2 = width // 2
    shapes = {(3, w2, 3, S), (w2, w2, 3, S // 2), (w2, width, 3, S // 2)}
    inplanes, H = width, S // 4
    for s in range(4):
        planes = width << s
        for i in range(2):
            stride = 2 if (i == 0 and s > 0) else 1
            shapes.add((inplanes, planes, 1, H))
            shapes.add((planes, planes, 3, H))
            H //= stride
            shapes.add((planes, 4 * planes, 1, H))
            if i == 0:
                shapes.add((inplanes, 4 * planes, 1, H))
            inplanes = 4 * planes
    return shapes


WIDE = {"RN50x4": (80, 288), "RN50x16": (96, 384), "RN50x64": (128, 448)}
CONV_SHAPES = sorted(set().union(*(_conv_shapes(w, S) for w, S in WIDE.values())))


@pytest.mark.parametrize("cin,cout,k,H", CONV_SHAPES)
def test_wide_conv2d_matches_torch(gpu_required, cin, cout, k, H):
    from marqo_b200.engine import debug_conv2d
    g = torch.Generator().manual_seed(cin * 7 + cout + k + H)
    n = 1 if H >= 96 else 3
    x = torch.randn(n, H, H, cin, generator=g)
    if cin != 3:
        x = torch.relu(x)
    w = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    b = torch.randn(cout, generator=g) * 0.1
    Ho = H // 2 if cin == 3 else H
    xd, wd = K.bf16(x).cuda().double(), K.bf16(w).cuda().double()
    conv = torch.nn.functional.conv2d(xd.permute(0, 3, 1, 2), wd, stride=2 if cin == 3 else 1, padding=k // 2)
    conv = conv.permute(0, 2, 3, 1) + b.cuda().double()
    scale = float(conv.abs().max())
    cases = [(True, None)]
    if k == 1 or cin == 3:
        cases.append((False, None))
    if cin != 3:
        cases.append((True, torch.randn(n, Ho, Ho, cout, generator=g)))
    for relu, res in cases:
        got = torch.from_numpy(debug_conv2d(x.numpy(), w.numpy(), b.numpy(), None if res is None else res.numpy(),
                                            relu=relu)).cuda()
        ref = conv + (K.bf16(res).cuda().double() if res is not None else 0)
        if relu:
            ref = torch.relu(ref)
        assert torch.isfinite(got).all()
        torch.testing.assert_close(got.double(), ref, rtol=2 ** -7, atol=1e-3 * scale)


@pytest.mark.parametrize("cin", [40, 48])
def test_conv3x3_halo_at_narrow_cin(gpu_required, cin):
    """A single 1 at each corner and edge midpoint of a 7 x 7 image: with cin < 64 a k-block spans taps, and the
    taps that fall outside the image must still read zeros on all four borders."""
    from marqo_b200.engine import debug_conv2d
    cout, H = cin, 7
    x = np.zeros((2, H, H, cin), np.float32)
    for y, xx in ((0, 0), (0, 6), (6, 0), (6, 6), (0, 3), (3, 0), (6, 3), (3, 6)):
        x[1, y, xx, :] = 1.0
    w = np.random.default_rng(cin).standard_normal((cout, cin, 3, 3)).astype(np.float32)
    got = debug_conv2d(x, w, relu=True)
    ref = torch.relu(torch.nn.functional.conv2d(torch.from_numpy(x).permute(0, 3, 1, 2).double(),
                                                K.bf16(torch.from_numpy(w)).double(), padding=1).permute(0, 2, 3, 1))
    assert not got[0].any()
    torch.testing.assert_close(torch.from_numpy(got).double(), ref, rtol=2 ** -7, atol=1e-2)


# ------------------------------------------------------------------------------------------------------------------
# The towers through the C ABI against the fp32 oracles
# ------------------------------------------------------------------------------------------------------------------
def _text_cfg(a):
    t = {k: a[k] for k in ("width", "layers", "heads", "mlp", "ctx", "vocab")} if "text" not in a else a["text"]
    return E.ClipCfg(embed_dim=a["embed_dim"], vision=E.TowerCfg(64, 1, 1, 64),
                     text=E.TowerCfg(t["width"], t["layers"], t["heads"], t["mlp"], ctx=t["ctx"], vocab=t["vocab"]),
                     act=a["act"])


def _check_text(enc, a, sd):
    ids = K.clip_text_ids(6, 7)
    tsd = {k: torch.as_tensor(v) for k, v in sd.items() if not k.startswith("visual.")}
    K.assert_embeddings_match(enc.encode_tokens(ids.numpy())[[0, 5]], E.clip_encode_text(tsd, _text_cfg(a), ids[[0, 5]]))


@pytest.mark.parametrize("name", ["RN50x16", "RN50x64", "RN50x4"])
def test_wide_resnet_towers(gpu_required, name):
    from marqo_b200.engine import Encoder
    a = _arch(name)
    S = a["resnet"]["image_size"]
    sd = _wide_weights(a, S)
    enc = Encoder("clip_resnet", a, sd, max_batch=8)
    try:
        assert enc.image_size == S
        rng = np.random.default_rng(S)
        at_size = rng.integers(0, 256, (8, S, S, 3), dtype=np.uint8)
        photo = rng.integers(0, 256, (3, 300, 517, 3), dtype=np.uint8)
        K.check_image_input_paths(enc, at_size, photo, lambda u8: E.clip_preprocess_u8(u8, S),
                                  lambda chw, normalize: O.encode_image(sd, a, chw.cuda(), normalize).cpu(),
                                  rows=[0, 7])
        _check_text(enc, a, sd)
    finally:
        enc.close()


def test_vit_l_14_336px_tower(gpu_required):
    from marqo_b200.engine import Encoder
    from marqo_b200.weights import random_clip_weights
    a = _arch("ViT-L/14@336px")
    sd = random_clip_weights(a, seed=336)
    enc = Encoder("clip", a, sd, max_batch=8)
    try:
        cfg = BV.clip_cfg(a)
        tsd = {k: torch.as_tensor(v).cuda() for k, v in sd.items() if k.startswith("visual.")}
        rng = np.random.default_rng(336)
        at_size = rng.integers(0, 256, (8, 336, 336, 3), dtype=np.uint8)
        photo = rng.integers(0, 256, (3, 400, 333, 3), dtype=np.uint8)
        K.check_image_input_paths(enc, at_size, photo, lambda u8: E.clip_preprocess_u8(u8, 336),
                                  lambda chw, normalize: E.clip_encode_image(tsd, cfg, chw.cuda(), normalize).cpu(),
                                  rows=[0, 7])
        _check_text(enc, a, sd)
    finally:
        enc.close()


# ------------------------------------------------------------------------------------------------------------------
# Through vectorise: the same network under both names, fp16, index and search
# ------------------------------------------------------------------------------------------------------------------
TWINS = {"ViT-B/32": "open_clip/ViT-B-32/openai", "ViT-B/16": "open_clip/ViT-B-16/openai",
         "ViT-L/14": "open_clip/ViT-L-14/openai", "RN50": "open_clip/RN50/openai", "RN101": "open_clip/RN101/openai"}


def _vectorise(name, content, modality, seed=31):
    from marqo_b200 import model_registry as R, s2_inference as s2
    tok = lambda texts: K.clip_text_ids(len(texts), len(texts[0])).numpy()
    props = dict(R.get_model_properties(name), random_init=seed, tokenizer=tok)
    s2.clear_loaded_models()
    try:
        return s2.vectorise(name, content, model_properties=props, device="cuda:0", normalize_embeddings=True,
                            modality=modality)
    finally:
        s2.clear_loaded_models()


@pytest.fixture(scope="module")
def photos():
    rng = np.random.default_rng(9)
    return [rng.integers(0, 256, (int(h), int(w), 3), dtype=np.uint8)
            for h, w in zip(rng.integers(150, 500, 6), rng.integers(150, 500, 6))]


@pytest.mark.parametrize("name", sorted(TWINS))
def test_clip_names_equal_their_open_clip_twins(gpu_required, photos, name):
    from marqo_b200.s2_inference import Modality
    texts = ["a photo of a dog", "a diagram"]
    for content, modality in ((photos, Modality.IMAGE), (texts, Modality.TEXT)):
        got = np.asarray(_vectorise(name, content, modality), np.float32)
        twin = np.asarray(_vectorise(TWINS[name], content, modality), np.float32)
        assert got.shape == twin.shape and np.isfinite(got).all()
        np.testing.assert_array_equal(got, twin)
        if name.startswith("ViT"):
            half = np.asarray(_vectorise("fp16/" + name, content, modality), np.float64)
            np.testing.assert_array_equal(half, got.astype(np.float16).astype(np.float64))


def test_fp16_loader_returns_float16(gpu_required, photos):
    from marqo_b200 import model_registry as R
    from marqo_b200.loaders import B200Clip, B200Fp16Clip
    p16 = dict(R.get_model_properties("fp16/ViT-B/32"), random_init=3)
    p32 = dict(R.get_model_properties("ViT-B/32"), random_init=3)
    m16, m32 = B200Fp16Clip(device="cuda:0", model_properties=p16), B200Clip(device="cuda:0", model_properties=p32)
    try:
        got, ref = m16.encode(photos[:3]), m32.encode(photos[:3])
        assert got.dtype == np.float16 and ref.dtype == np.float32
        np.testing.assert_array_equal(got, ref.astype(np.float16))
        dev = m16.encode_to_device(photos[:3], default="image")
        np.testing.assert_array_equal(dev.cpu().numpy(), ref.astype(np.float16).astype(np.float32))
    finally:
        m16.close()
        m32.close()


def test_vectorise_custom_rn50x16_checkpoint_into_index_and_search(gpu_required, score_oracle, photos, tmp_path):
    """A custom `clip` model from an RN50x16 checkpoint file without an arch (the loader reads it from the shapes)."""
    from marqo_b200 import s2_inference as s2
    from marqo_b200.s2_inference import Modality
    path = tmp_path / "RN50x16.npz"
    np.savez(path, **_wide_weights(_arch("RN50x16"), 16))
    props = {"name": "my-rn50x16", "type": "clip", "dimensions": 768, "localpath": str(path)}
    rng = np.random.default_rng(16)
    images = photos + [rng.integers(0, 256, (384, 384, 3), dtype=np.uint8) for _ in range(10)]
    s2.clear_loaded_models()
    try:
        docs = np.asarray(s2.vectorise("my-rn50x16", images, model_properties=props, device="cuda:0",
                                       normalize_embeddings=True, modality=Modality.IMAGE), np.float32)
        queries = np.asarray(s2.vectorise("my-rn50x16", images[:3], model_properties=props, device="cuda:0",
                                          normalize_embeddings=True, modality=Modality.IMAGE), np.float32)
    finally:
        s2.clear_loaded_models()
    assert docs.shape == (16, 768)
    K.assert_index_search_matches(score_oracle, docs, queries)


@pytest.mark.parametrize("S", [288, 384, 448])
def test_resize_matches_pillow_at_the_wide_resnet_sizes(gpu_required, S):
    """The wide ResNets crop to 288, 384 and 448, sizes no registered model uses: the resize there against Pillow's
    Resize(S, BICUBIC) + CenterCrop(S), bit for bit."""
    from PIL import Image
    from torchvision.transforms import CenterCrop, InterpolationMode, Resize
    from marqo_b200.engine import debug_resize
    for h, w in ((480, 640), (S, 1000), (S + 1, 333), (1000, 50)):
        imgs = np.random.default_rng(h * 7 + w).integers(0, 256, (2, h, w, 3), dtype=np.uint8)
        ref = []
        for a in imgs:
            im = Image.fromarray(a)
            for t in (Resize(S, interpolation=InterpolationMode.BICUBIC), CenterCrop(S)):
                im = t(im)
            ref.append(np.asarray(im.convert("RGB")))
        np.testing.assert_array_equal(debug_resize(imgs, S), np.stack(ref), err_msg=f"S = {S}, {h} x {w}")


# ------------------------------------------------------------------------------------------------------------------
# RN50's output against a library built from an earlier commit (MARQO_B200_BASELINE_LIB), in the same GPU session
# ------------------------------------------------------------------------------------------------------------------
_RN50_SCRIPT = """
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from marqo_b200 import model_registry as R
from marqo_b200.engine import Encoder
from marqo_b200.weights import random_clip_resnet_weights
a = R.get_model_properties("open_clip/RN50/openai")["arch"]
enc = Encoder("clip_resnet", a, random_clip_resnet_weights(a, seed=77), max_batch=32)
img = np.random.default_rng(77).integers(0, 256, (32, 224, 224, 3), dtype=np.uint8)
np.save(sys.argv[2], enc.encode_images_u8(img))
enc.close()
"""


@pytest.mark.skipif(not os.environ.get("MARQO_B200_BASELINE_LIB"), reason="no baseline library to compare against")
def test_rn50_output_unchanged_against_baseline_library(gpu_required, tmp_path):
    """RN50 (power-of-two channels only) through a library built from an earlier commit and through this one, each in
    its own process on the same GPU: the same bits.  Build the baseline with
        git worktree add /tmp/base <commit> && (cd /tmp/base && python -m marqo_b200.build)
    copy /tmp/base/marqo_b200/libmarqo_b200.so to an ignored path inside the tree (*.so is ignored) and name it in
    MARQO_B200_BASELINE_LIB.  A checkout has no earlier commit's sources to build from, so without one it skips."""
    outs = []
    for lib in (os.environ["MARQO_B200_BASELINE_LIB"], None):
        env = dict(os.environ)
        env.pop("MARQO_B200_LIB", None)
        if lib:
            env["MARQO_B200_LIB"] = lib
        out = tmp_path / f"rn50_{len(outs)}.npy"
        subprocess.run([sys.executable, "-c", _RN50_SCRIPT, str(ROOT), str(out)], env=env, check=True, timeout=600)
        outs.append(np.load(out))
    assert np.isfinite(outs[1]).all()
    np.testing.assert_array_equal(outs[1], outs[0])
