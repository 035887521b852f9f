"""OWL-ViT detection end to end on the H100: the full-depth B/32 forward, and B/16 and L/14 at two layers with their
full token counts, against the fp32 oracle (tests/_owlvit_oracle.py) on 240 x 240 images squashed by Pillow; the
refusals; launch counts and graph replay; device memory after destroy; and the served ReRankerOwl subclass against the
oracle-driven reference loop."""
import numpy as np
import pytest
import torch

import _owlvit_oracle as O
from marqo_b200 import _native as N

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available(), reason="needs an H100 (sm_90a)")]

# Bounds on |engine - oracle| for the logits (absolute, plus a share of |logit|) and the boxes (absolute), above the
# largest differences measured on the H100 (DESIGN.md §7.5s).
LOGIT_ATOL, LOGIT_RTOL, BOX_ATOL = 0.1, 0.01, 0.005


def _arch(name, layers=None):
    from marqo_b200 import model_registry as R
    a = R.OWL_VIT_MODELS[name]["arch"]
    if layers is None:
        return a
    return {**a, "vision": {**a["vision"], "layers": layers}, "text": {**a["text"], "layers": layers}}


def _squash(imgs, S):
    from test_ragged_images_gpu import _pillow
    return np.stack([_pillow(a, S, True) for a in imgs])


def _query():
    ids = np.zeros(16, np.int32)
    ids[:6] = [49406, 320, 1929, 539, 320, 49407]
    return ids


@pytest.fixture(scope="module")
def b32():
    from marqo_b200 import weights as W
    from marqo_b200.engine import Encoder
    arch = _arch("owl/ViT-B/32")
    sd = W.random_owlvit_weights(arch, 21)
    enc = Encoder("clip", arch, W.owlvit_state_dict_to_engine(sd), max_batch=8)
    yield arch, sd, enc
    enc.close()


def _compare(arch, sd, enc, imgs, what):
    ids = _query()
    logits, boxes = enc.detect_images_u8(imgs, ids)
    S = arch["vision"]["image_size"]
    rl, rb = O.detect(sd, O.pixels_from_u8(_squash(imgs, S)), torch.from_numpy(ids).long(),
                      arch["vision"]["heads"], arch["text"]["heads"])
    rl, rb = rl.numpy(), rb.numpy()
    le, be = np.abs(logits - rl), np.abs(boxes - rb)
    print(f"\n[owl {what}] max |logit err| {le.max():.4g} (|logit| up to {np.abs(rl).max():.3g}), "
          f"max |box err| {be.max():.4g}")
    assert np.isfinite(logits).all() and np.isfinite(boxes).all()
    assert (le <= LOGIT_ATOL + LOGIT_RTOL * np.abs(rl)).all()
    assert (be <= BOX_ATOL).all()
    for i in range(len(imgs)):
        top2 = np.sort(rl[i])[-2:]
        if top2[1] - top2[0] > 2 * (LOGIT_ATOL + LOGIT_RTOL * abs(top2[1])):
            assert int(np.argmax(logits[i])) == int(np.argmax(rl[i])), f"{what}: image {i} top box"


def _images(n, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, 240, 240, 3), dtype=np.uint8)


def test_b32_full_depth_matches_oracle(b32):
    arch, sd, enc = b32
    _compare(arch, sd, enc, _images(3, 1), "B/32 full depth")


@pytest.mark.parametrize("name", ["owl/ViT-B/16", "owl/ViT-L/14"])
def test_reduced_depth_matches_oracle(gpu_required, name):
    from marqo_b200 import weights as W
    from marqo_b200.engine import Encoder
    arch = _arch(name, layers=2)
    sd = W.random_owlvit_weights(arch, 22)
    enc = Encoder("clip", arch, W.owlvit_state_dict_to_engine(sd), max_batch=2)
    try:
        _compare(arch, sd, enc, _images(2, 3), f"{name} 2 layers")
    finally:
        enc.close()


def test_sub_batches_and_graph_replay(b32):
    """n over max_batch runs in sub-batches; repeated calls (eager, captured, replayed) give identical bits and
    launch counts, and each image's result does not depend on its neighbours."""
    arch, sd, enc = b32
    imgs = _images(11, 5)
    runs = [enc.detect_images_u8(imgs, _query()) for _ in range(3)]
    launches = []
    for _ in range(3):
        enc.detect_images_u8(imgs[:2], _query())
        launches.append(enc.last_timing()[1])
    for lg, bx in runs[1:]:
        assert np.array_equal(lg, runs[0][0]) and np.array_equal(bx, runs[0][1])
    lg1, bx1 = enc.detect_images_u8(imgs[9:10], _query())
    assert np.array_equal(lg1[0], runs[0][0][9]) and np.array_equal(bx1[0], runs[0][1][9])
    layers = arch["vision"]["layers"] + arch["text"]["layers"]
    assert launches[0] == launches[1] == launches[2]
    # per call: the text tower (embed, 7 per layer, the two-kernel head) and, per sub-batch, the two-pass resize, the
    # trunk (embed, patch GEMM, ln_pre, 7 per layer), the merge, the 3 head GEMMs, logits and boxes
    assert launches[0] == 7 * layers + 14, launches


def test_refusals(b32):
    from _checks import assert_refused
    from marqo_b200 import weights as W
    from marqo_b200.engine import Encoder
    arch, sd, enc = b32
    imgs = _images(1, 0)
    for call in (lambda: enc.encode_images_u8(imgs), lambda: enc.encode_tokens(_query()[None]),
                 lambda: enc.detect_images_u8(imgs, np.zeros(17, np.int32)),
                 lambda: enc.detect_images_u8(imgs[:0], _query()),
                 lambda: enc.detect_images_u8(np.zeros((1, 0, 240, 3), np.uint8), _query())):
        with pytest.raises(N.NativeError) as e:
            call()
        assert e.value.code == N.ERR_INVALID_ARG, e.value
    small = _arch("owl/ViT-B/32", layers=1)
    eng = W.owlvit_state_dict_to_engine(W.random_owlvit_weights(small, 2))
    plain = {**small, "owl_detect": False}
    clip_sd = {**eng, "visual.proj": np.zeros((768, 512), np.float32)}
    e2 = Encoder("clip", plain, clip_sd, max_batch=1)
    try:
        with pytest.raises(N.NativeError) as e:
            e2.detect_images_u8(imgs, _query())
        assert e.value.code == N.ERR_INVALID_ARG
    finally:
        e2.close()
    for missing in ("layer_norm.weight", "class_head.logit_scale.bias", "box_head.dense2.weight"):
        assert_refused("clip", small, {k: v for k, v in eng.items() if k != missing}, N.ERR_MISSING_WEIGHT, missing)
    assert_refused("clip", {**small, "resize_mode": "crop"}, eng, N.ERR_INVALID_ARG, "squash")
    bert = {"width": 128, "layers": 1, "heads": 2, "mlp": 256, "vocab": 100, "max_pos": 16}
    d = N.ModelDesc()
    d.arch, d.max_batch, d.embed_dim, d.owl_detect = N.ARCH_BERT, 1, 128, 1
    d.text = N.TowerDesc(bert["width"], 1, 2, 256, 16, 100, 0, 0)
    import ctypes as C
    h = C.c_void_p()
    assert N.load().b200_model_create(0, C.byref(d), C.byref(h)) == N.ERR_INVALID_ARG


def test_device_memory_returns_after_destroy(gpu_required):
    from marqo_b200 import weights as W
    from marqo_b200.engine import Encoder
    arch = _arch("owl/ViT-B/32", layers=1)
    eng = W.owlvit_state_dict_to_engine(W.random_owlvit_weights(arch, 4))
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    enc = Encoder("clip", arch, eng, max_batch=4)
    enc.detect_images_u8(_images(5, 9), _query())
    enc.close()
    torch.cuda.synchronize()
    assert abs(torch.cuda.mem_get_info()[0] - free0) <= (8 << 20)


class _EngineOracle:
    """The oracle behind the detect surface, with the engine's squash done by Pillow."""

    def __init__(self, arch, sd, ids):
        self.arch, self.sd, self.ids = arch, sd, ids

    def raw(self, images):
        hwc = _squash(np.stack([np.asarray(im) for im in images]), self.arch["vision"]["image_size"])
        return O.detect(self.sd, O.pixels_from_u8(hwc), torch.from_numpy(self.ids).long(),
                        self.arch["vision"]["heads"], self.arch["text"]["heads"])

    def detect(self, query, images):
        logits, boxes = self.raw(images)
        return [O.post_process(logits[i], boxes[i], 240, 240) for i in range(len(images))]


def test_served_reranker_end_to_end(b32, tmp_path):
    """The served subclass with B200OwlDetector (seeded weights) against the same subclass driven by the oracle: the
    same top box per hit wherever the oracle separates them, scores within the logit bound through the sigmoid."""
    from oracle import tokenizers as OT
    from test_owlvit import _StandOwl, _helpers
    from marqo_b200.owl_reranker import B200OwlDetector, make_owl_reranker_class
    from PIL import Image
    arch, sd, _ = b32
    merges = OT.train_toy_merges(["a photo of a cat", "a cat on a mat"] * 3, 50)
    (tmp_path / "merges.txt").write_text(merges)
    det = B200OwlDetector("owl/ViT-B/32", device="cuda", weights=sd, merges_file=str(tmp_path / "merges.txt"))
    try:
        ids = det.query_ids("a cat")
        imgs = [Image.fromarray(a) for a in _images(4, 17)]
        sizes = [(300, 200), (640, 480), (240, 240), (1000, 90)]
        _StandOwl.images, _StandOwl.sizes = imgs, sizes
        cls = make_owl_reranker_class(_StandOwl, _helpers(), None)
        got, want = cls("owl/ViT-B/32", "cuda", (240, 240)), cls("owl/ViT-B/32", "cuda", (240, 240))
        got.model, want.model = det, _EngineOracle(arch, sd, ids)
        for r in (got, want):
            r.rerank("a cat", {"hits": [{} for _ in imgs]}, ["image"], num_highlights=1)
        sg, sw = got.scores.double(), want.scores.double()
        assert ((sg - sw).abs() <= 0.25 * (LOGIT_ATOL + LOGIT_RTOL * 20)).all()
        rl, _ = want.model.raw(imgs)
        for i in range(len(imgs)):
            top2 = np.sort(rl[i].numpy())[-2:]
            if top2[1] - top2[0] > 2 * (LOGIT_ATOL + LOGIT_RTOL * abs(top2[1])):
                torch.testing.assert_close(got.boxes[i], want.boxes[i], rtol=0, atol=BOX_ATOL * 240 * 2)
                assert got.boxes_original[i] == pytest.approx(want.boxes_original[i], abs=BOX_ATOL * 1000 * 2)
        assert got.identifier == want.identifier
    finally:
        det.close()
