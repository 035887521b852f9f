"""Every model call of the C ABI on one small model of every kind, through the raw library: which calls each model
takes (a refused call returns ERR_INVALID_ARG, writes nothing on the host or the device and leaves last_timing as it
was), the argument refusals of each call in both forms, the host form of a call against its device form bit for bit
and launch for launch within one sub-batch and across several, and every accepted call's outputs against a baseline
library built from an earlier commit."""
import copy
import ctypes as C
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import _coca_oracle as CO
import _cross_encoder_oracle as CE
import _eva02_oracle as V
import _mclip_oracle as MC
import _mpnet_oracle as MP
import _siglip_oracle as SO
import _xlmr_oracle as X
from marqo_b200 import _native as N
from oracle import encoders as E

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
MAX_BATCH = 2   # the sub-batch of every call: n = 3 takes two

IMAGE_CALLS = ["images_u8", "images_u8_device", "images_u8_ragged", "images_u8_ragged_device", "images_f32"]
CALLS = IMAGE_CALLS + ["tokens", "tokens_device", "classify", "classify_device", "detect", "videos", "videos_device"]
# the device form of every call that has one
DEVICE_FORM = {"images_u8": "images_u8_device", "images_u8_ragged": "images_u8_ragged_device",
               "tokens": "tokens_device", "classify": "classify_device", "videos": "videos_device"}
IMAGES, TOKENS, CLASSIFY = set(IMAGE_CALLS), {"tokens", "tokens_device"}, {"classify", "classify_device"}
DETECT, VIDEOS = {"detect"}, {"videos", "videos_device"}


def _tower(t):
    return dict(width=t.width, layers=t.layers, heads=t.heads, mlp=t.mlp, ctx=t.ctx, vocab=t.vocab,
                image_size=t.image_size, patch=t.patch)


def _clip():
    cfg = E.tiny_clip("quickgelu")
    arch = dict(embed_dim=cfg.embed_dim, act=cfg.act, mean=cfg.mean, std=cfg.std, vision=_tower(cfg.vision),
                text=_tower(cfg.text))
    return "clip", arch, E.make_clip_weights(cfg, seed=1)


def _siglip():
    cfg = SO.tiny_siglip()
    return "siglip", cfg.arch(), SO.make_siglip_weights(cfg, seed=2)


def _resnet():
    from marqo_b200.weights import random_clip_resnet_weights
    arch = dict(embed_dim=128, act="quickgelu", mean=E.OPENAI_CLIP_MEAN, std=E.OPENAI_CLIP_STD, width=128, layers=1,
                heads=2, mlp=512, ctx=77, vocab=1000, resnet=dict(layers=[1, 1, 1, 1], width=64, heads=32))
    return "clip_resnet", arch, random_clip_resnet_weights(arch, seed=3)


def _convnext():
    from marqo_b200 import model_registry as R
    from marqo_b200.weights import random_clip_convnext_weights
    arch = R.get_model_properties("open_clip/convnext_base_w/laion2b_s13b_b82k")["arch"]
    arch["convnext"]["depths"], arch["layers"] = [1, 1, 1, 1], 0
    return "clip_convnext", arch, random_clip_convnext_weights(arch, seed=4)


def _eva02():
    from marqo_b200.weights import random_eva02_weights
    arch = V.arch(V.B16, eva_layers=1, text_layers=1)
    return "clip_eva", arch, random_eva02_weights(arch, seed=5)


def _coca():
    a = CO.arch(CO.NAMES[0], vision_layers=1, text_layers=1)
    return "clip", a, CO.weights(a, 6)


def _owlvit():
    from marqo_b200 import model_registry as R
    from marqo_b200 import weights as W
    a = copy.deepcopy(R.OWL_VIT_MODELS["owl/ViT-B/32"]["arch"])
    a["vision"]["layers"] = a["text"]["layers"] = 1
    return "clip", a, W.owlvit_state_dict_to_engine(W.random_owlvit_weights(a, 7))


def _languagebind():
    from marqo_b200 import model_registry as R
    from marqo_b200 import weights as W
    a = copy.deepcopy(R.LANGUAGEBIND_MODELS["LanguageBind/Video_V1.5_FT"]["arch"])
    a["vision"]["layers"] = a["text"]["layers"] = 1
    return "clip", a, W.languagebind_video_state_dict_to_engine(W.random_languagebind_video_weights(a, 8))


def _bert():
    cfg = E.tiny_bert("mean")
    arch = dict(width=cfg.width, layers=cfg.layers, heads=cfg.heads, mlp=cfg.mlp, vocab=cfg.vocab, max_pos=cfg.max_pos,
                type_vocab=cfg.type_vocab, pool=cfg.pool)
    return "bert", arch, E.make_bert_weights(cfg, seed=9)


def _cross_encoder():
    a = CE.arch("cross-encoder/ms-marco-TinyBERT-L-2", layers=1)
    return "bert", a, CE.weights(a, 10)


def _mclip():
    a = MC.arch("multilingual-clip/XLM-Roberta-Large-Vit-B-32", layers=1, vocab=1000)
    return a["text_kind"], a, MC.text_weights(a, 11)


def _mpnet():
    cfg = MP.tiny_mpnet()
    return "mpnet", MP.engine_config(cfg), MP.make_mpnet_weights(cfg, seed=12)


def _xlmr():
    cfg = X.tiny_xlmr()
    return "xlmr", X.engine_config(cfg), X.make_xlmr_weights(cfg, seed=13)


def _gte():
    from marqo_b200 import model_registry as R
    from marqo_b200.weights import random_gte_weights
    arch = dict(R.get_model_properties("Marqo/dunzhang-stella_en_400M_v5")["arch"], layers=1)
    return "gte", arch, random_gte_weights(arch, seed=14)


# name: (builder, the ids per sequence of its token calls, the calls it takes)
MODELS = {
    "clip_vit": (_clip, 16, IMAGES | TOKENS),
    "siglip": (_siglip, 16, IMAGES | TOKENS),
    "resnet": (_resnet, 16, IMAGES | TOKENS),
    "convnext": (_convnext, 16, IMAGES),
    "eva02": (_eva02, 16, IMAGES | TOKENS),
    "coca": (_coca, CO.TEXT_IDS, IMAGES | TOKENS),
    "owlvit": (_owlvit, 12, DETECT),
    "languagebind": (_languagebind, 16, VIDEOS | TOKENS),
    "bert": (_bert, 16, TOKENS),
    "cross_encoder": (_cross_encoder, 16, CLASSIFY),
    "mclip": (_mclip, 16, TOKENS),
    "mpnet": (_mpnet, 16, TOKENS),
    "xlmr": (_xlmr, 16, TOKENS),
    "gte": (_gte, 16, TOKENS),
}


def _encoder(name):
    from marqo_b200.engine import Encoder
    kind, arch, sd = MODELS[name][0]()
    return Encoder(kind, arch, sd, max_batch=MAX_BATCH)


class _Inputs:
    """Seeded inputs of every call for n items, on the host and the device (images of a size the tower resizes)."""

    def __init__(self, enc, seq, n, seed):
        rng = np.random.default_rng(seed)
        S = enc.image_size or 32
        self.n, self.seq, self.hw, self.frames = n, seq, (S + 6, S - 10), getattr(enc, "video_frames", 0) or 2
        self.img = rng.integers(0, 256, (n,) + self.hw + (3,), dtype=np.uint8)
        sizes = [(S, S), (S // 2, S + 7), (S + 6, S - 10)]
        self.ragged = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in sizes[:n]]
        self.chw = rng.standard_normal((n, 3, S, S)).astype(np.float32)
        self.ids = rng.integers(5, 100, (n, seq)).astype(np.int32)
        lens = [seq] + list(rng.integers(2, seq + 1, n - 1))
        self.mask = (np.arange(seq)[None, :] < np.array(lens)[:, None]).astype(np.int32)
        self.types = (np.arange(seq)[None, :] >= seq // 2).astype(np.int32) * self.mask
        self.video = rng.integers(0, 256, (n, self.frames, 30, 40, 3), dtype=np.uint8)
        cuda = lambda a: torch.from_numpy(a).cuda()
        self.d_img, self.d_chw, self.d_video = cuda(self.img), cuda(self.chw), cuda(self.video)
        self.d_ragged = [cuda(a) for a in self.ragged]
        self.d_ids, self.d_mask, self.d_types = cuda(self.ids), cuda(self.mask), cuda(self.types)
        self.hs = np.array([a.shape[0] for a in self.ragged], np.int32)
        self.ws = np.array([a.shape[1] for a in self.ragged], np.int32)
        P = getattr(enc, "grid", 0) ** 2 or 1
        self.emb = np.full((n, enc.embed_dim), np.nan, np.float32)
        self.d_emb = torch.full((n, enc.embed_dim), float("nan"), device="cuda")
        self.logits = np.full((n, P), np.nan, np.float32)
        self.boxes = np.full((n, P, 4), np.nan, np.float32)
        torch.cuda.synchronize()

    def outputs(self, call):
        """The outputs `call` writes, as host arrays."""
        if call == "detect":
            return [self.logits.copy(), self.boxes.copy()]
        return [self.d_emb.cpu().numpy() if call.endswith("_device") else self.emb.copy()]

    def untouched(self):
        return (np.isnan(self.emb).all() and bool(torch.isnan(self.d_emb).all()) and np.isnan(self.logits).all()
                and np.isnan(self.boxes).all())


def _call(lib, enc, call, x, null=None, n=None, seq=None, frames=None, act=1, mask=None):
    """Make `call` on enc through the raw library over inputs x; null names the buffer passed as NULL ("in", "out",
    "query", "boxes", "heights", "widths", "entry": one image of a ragged call); the keywords replace an argument."""
    h = enc._handle()
    n = x.n if n is None else n
    seq = x.seq if seq is None else seq
    frames = x.frames if frames is None else frames
    mask = x.mask if mask is None else mask
    hp = lambda key, a: None if null == key else a.ctypes.data_as(C.c_void_p)
    dp = lambda key, t: None if null == key else C.c_void_p(t.data_ptr())
    H, W = x.hw
    if call == "images_u8":
        return lib.b200_model_encode_images_u8(h, hp("in", x.img), n, H, W, 1, hp("out", x.emb))
    if call == "images_u8_device":
        return lib.b200_model_encode_images_u8_device(h, dp("in", x.d_img), n, H, W, 1, dp("out", x.d_emb), 1)
    if call in ("images_u8_ragged", "images_u8_ragged_device"):
        device = call.endswith("_device")
        ptrs = [t.data_ptr() for t in x.d_ragged] if device else [a.ctypes.data for a in x.ragged]
        if null == "entry":
            ptrs[-1] = None
        arr = None if null == "in" else (C.c_void_p * len(ptrs))(*ptrs)
        if device:
            return lib.b200_model_encode_images_u8_ragged_device(h, arr, hp("heights", x.hs), hp("widths", x.ws), n,
                                                                 1, dp("out", x.d_emb), 1)
        return lib.b200_model_encode_images_u8_ragged(h, arr, hp("heights", x.hs), hp("widths", x.ws), n, 1,
                                                      hp("out", x.emb))
    if call == "images_f32":
        return lib.b200_model_encode_images_f32(h, hp("in", x.chw), n, 1, hp("out", x.emb))
    if call == "tokens":
        return lib.b200_model_encode_tokens(h, hp("in", x.ids), hp("mask", mask), n, seq, 1, hp("out", x.emb))
    if call == "tokens_device":
        return lib.b200_model_encode_tokens_device(h, dp("in", x.d_ids), dp("mask", x.d_mask), n, seq, 1,
                                                   dp("out", x.d_emb), 1)
    if call == "classify":
        return lib.b200_model_classify_tokens(h, hp("in", x.ids), hp("mask", mask), hp("types", x.types), n, seq, act,
                                              hp("out", x.emb))
    if call == "classify_device":
        return lib.b200_model_classify_tokens_device(h, dp("in", x.d_ids), dp("mask", x.d_mask),
                                                     dp("types", x.d_types), n, seq, act, dp("out", x.d_emb), 1)
    if call == "detect":
        return lib.b200_model_detect_images_u8(h, hp("in", x.img), n, H, W, hp("query", x.ids[0]), seq,
                                               hp("out", x.logits), hp("boxes", x.boxes))
    if call == "videos":
        return lib.b200_model_encode_videos_u8(h, hp("in", x.video), n, frames, 30, 40, 1, hp("out", x.emb))
    assert call == "videos_device"
    return lib.b200_model_encode_videos_u8_device(h, dp("in", x.d_video), n, frames, 30, 40, 1, dp("out", x.d_emb), 1)


def _timing(lib, enc):
    ms, launches = C.c_float(0), C.c_int(0)
    rc = lib.b200_model_last_timing(enc._handle(), C.byref(ms), C.byref(launches))
    return rc, ms.value, launches.value


@pytest.fixture(scope="module", params=list(MODELS))
def model(request, gpu_required):
    enc = _encoder(request.param)
    yield request.param, enc
    enc.close()


def test_each_model_takes_its_calls_and_refuses_the_others(model):
    name, enc = model
    _, seq, takes = MODELS[name]
    lib = N.load()
    for call in sorted(takes):   # an accepted call first, so that there is a timing to keep
        assert _call(lib, enc, call, _Inputs(enc, seq, 2, 0)) == N.OK, (name, call, lib.b200_last_error())
    before = _timing(lib, enc)
    assert before[0] == N.OK
    for call in CALLS:
        if call in takes:
            continue
        x = _Inputs(enc, seq, 2, 0)
        assert _call(lib, enc, call, x) == N.ERR_INVALID_ARG, (name, call)
        torch.cuda.synchronize()
        assert x.untouched(), (name, call)
        assert _timing(lib, enc) == before, (name, call)


def _argument_refusals(call, x):
    """(what, keywords of _call) for every argument refusal of `call`, with the code each returns."""
    nulls = {"images_u8_ragged": ["in", "heights", "widths", "entry", "out"], "detect": ["in", "query", "out", "boxes"]}
    nulls["images_u8_ragged_device"] = nulls["images_u8_ragged"]
    cases = [(f"NULL {b}", dict(null=b), N.ERR_INVALID_ARG) for b in nulls.get(call, ["in", "out"])]
    cases += [("n = 0", dict(n=0), N.ERR_INVALID_ARG), ("n < 0", dict(n=-1), N.ERR_INVALID_ARG)]
    if call in TOKENS | CLASSIFY | DETECT:
        cases += [("seq = 0", dict(seq=0), N.ERR_INVALID_ARG), ("seq too long", dict(seq=100000), N.ERR_INVALID_ARG)]
    if call in VIDEOS:
        cases += [("frames - 1", dict(frames=x.frames - 1), N.ERR_INVALID_ARG),
                  ("frames + 1", dict(frames=x.frames + 1), N.ERR_INVALID_ARG)]
    if call in CLASSIFY:
        cases += [("activation 2", dict(act=2), N.ERR_INVALID_ARG), ("activation -1", dict(act=-1), N.ERR_INVALID_ARG)]
    if call in ("tokens", "classify"):
        holes = x.mask.copy()
        holes[0, 1] = 0   # a zero before ones: not a prefix mask
        cases.append(("mask with a hole", dict(mask=holes), N.ERR_UNSUPPORTED))
    return cases


def test_argument_refusals_write_nothing(model):
    name, enc = model
    _, seq, takes = MODELS[name]
    lib = N.load()
    for call in sorted(takes):
        for what, kw, code in _argument_refusals(call, _Inputs(enc, seq, 2, 0)):
            if name in ("clip_vit", "resnet", "eva02", "coca", "languagebind") and what == "mask with a hole":
                continue   # causal text towers take any mask
            x = _Inputs(enc, seq, 2, 0)
            assert _call(lib, enc, call, x, **kw) == code, (name, call, what)
            torch.cuda.synchronize()
            assert x.untouched(), (name, call, what)


@pytest.mark.parametrize("n", [MAX_BATCH, MAX_BATCH + 1], ids=["one sub-batch", "two sub-batches"])
def test_host_form_equals_device_form(model, n):
    name, enc = model
    _, seq, takes = MODELS[name]
    lib = N.load()
    for host, device in DEVICE_FORM.items():
        if host not in takes:
            continue
        got = {}
        for call in (host, device):
            x = _Inputs(enc, seq, n, 1)
            assert _call(lib, enc, call, x) == N.OK, (name, call, lib.b200_last_error())
            got[call] = (x.outputs(call)[0], _timing(lib, enc)[2])
        assert np.isfinite(got[host][0]).all(), (name, host)
        np.testing.assert_array_equal(got[device][0], got[host][0], err_msg=f"{name}: {host}")
        assert got[device][1] == got[host][1], (name, host, "launches")


def _outputs_of_every_accepted_call(out_path):
    """Run every accepted call of every model at n = MAX_BATCH + 1 on seeded inputs; save the outputs to out_path."""
    lib, saved = N.load(), {}
    for name, (_, seq, takes) in MODELS.items():
        enc = _encoder(name)
        try:
            for call in sorted(takes):
                x = _Inputs(enc, seq, MAX_BATCH + 1, 2)
                assert _call(lib, enc, call, x) == N.OK, (name, call, lib.b200_last_error())
                for i, a in enumerate(x.outputs(call)):
                    saved[f"{name}/{call}/{i}"] = a
        finally:
            enc.close()
    np.savez(out_path, **saved)


@pytest.mark.skipif(not os.environ.get("MARQO_B200_BASELINE_LIB"), reason="no baseline library to compare against")
def test_outputs_unchanged_against_baseline_library(gpu_required, tmp_path):
    """Every accepted call through a library built from an earlier commit and through this one, each in its own
    process on the same GPU: the same bits.  MARQO_B200_BASELINE_LIB names the baseline library, built as
    test_openai_clip_gpu.py::test_rn50_output_unchanged_against_baseline_library describes."""
    outs = []
    for lib in (os.environ["MARQO_B200_BASELINE_LIB"], None):
        env = dict(os.environ)
        env.pop("MARQO_B200_LIB", None)
        if lib:
            env["MARQO_B200_LIB"] = lib
        env["PYTHONPATH"] = os.pathsep.join([str(ROOT), str(ROOT / "tests"), env.get("PYTHONPATH", "")])
        out = tmp_path / f"calls_{len(outs)}.npz"
        script = f"import test_model_calls_gpu as T; T._outputs_of_every_accepted_call({str(out)!r})"
        subprocess.run([sys.executable, "-c", script], cwd=ROOT, env=env, check=True, timeout=1200)
        outs.append(dict(np.load(out)))
    assert sorted(outs[1]) == sorted(outs[0])
    for key in outs[0]:
        assert np.isfinite(outs[1][key]).all(), key
        np.testing.assert_array_equal(outs[1][key], outs[0][key], err_msg=key)
