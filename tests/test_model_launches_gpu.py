"""The launch count b200_model_last_timing reports, and the GEMM / attention launches b200_model_profile brackets, equal
the kernels the device ran (torch.profiler's CUDA kernel events) for one small model of every tower kind, through
every encode entry point, with and without L2 normalisation; and a replayed CUDA graph reports the count of the eager
pass it was captured from.  Served models at reduced depth report the count their layers add up to, with the
variant-specific kernels (rotary, SwiGLU, GeGLU, wgmma attention) run as often as the layers call them."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile

import _eva02_oracle as V
import _mpnet_oracle as M
import _siglip_oracle as O
import _xlmr_oracle as X
from oracle import encoders as E

pytestmark = pytest.mark.gpu
SEQ = 16


def _clip():
    cfg = E.tiny_clip("quickgelu")
    tower = lambda t: dict(width=t.width, layers=t.layers, heads=t.heads, mlp=t.mlp, ctx=t.ctx, vocab=t.vocab,
                           image_size=t.image_size, patch=t.patch)
    arch = dict(embed_dim=cfg.embed_dim, act=cfg.act, mean=cfg.mean, std=cfg.std, vision=tower(cfg.vision),
                text=tower(cfg.text))
    return "clip", arch, E.make_clip_weights(cfg, seed=1), cfg.text.vocab


def _siglip():
    cfg = O.tiny_siglip()
    return "siglip", cfg.arch(), O.make_siglip_weights(cfg, seed=2), cfg.vocab


def _clip_resnet():
    # the smallest ModifiedResNet the runtime takes, with the tiny CLIP text tower
    from marqo_b200.weights import random_clip_resnet_weights
    arch = dict(embed_dim=128, act="quickgelu", mean=E.OPENAI_CLIP_MEAN, std=E.OPENAI_CLIP_STD, width=128, layers=2,
                heads=2, mlp=512, ctx=77, vocab=1000, resnet=dict(layers=[1, 1, 1, 1], width=64, heads=32))
    return "clip_resnet", arch, random_clip_resnet_weights(arch, seed=3), 1000


def _clip_eva():
    from marqo_b200.weights import random_eva02_weights
    arch = V.arch(V.B16, eva_layers=1, text_layers=1)
    return "clip_eva", arch, random_eva02_weights(arch, seed=7), arch["vocab"]


def _bert():
    cfg = E.tiny_bert("mean")
    arch = dict(width=cfg.width, layers=cfg.layers, heads=cfg.heads, mlp=cfg.mlp, vocab=cfg.vocab, max_pos=cfg.max_pos,
                type_vocab=cfg.type_vocab, pool=cfg.pool)
    return "bert", arch, E.make_bert_weights(cfg, seed=4), cfg.vocab


def _mpnet():
    cfg = M.tiny_mpnet()
    return "mpnet", M.engine_config(cfg), M.make_mpnet_weights(cfg, seed=5), cfg.vocab


def _xlmr():
    cfg = X.tiny_xlmr()
    return "xlmr", X.engine_config(cfg), X.make_xlmr_weights(cfg, seed=6), cfg.vocab


def _gte():
    from marqo_b200 import model_registry as R
    from marqo_b200.weights import random_gte_weights
    arch = dict(R.get_model_properties("Marqo/dunzhang-stella_en_400M_v5")["arch"], layers=2)
    return "gte", arch, random_gte_weights(arch, seed=8), arch["vocab"]


def _kernels(fn):
    """Run fn under torch.profiler; the names of the CUDA kernels it ran (copies and memsets left out)."""
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    names = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA]
    return [n for n in names if not n.startswith(("Memcpy", "Memset"))]


def _base_name(kernel):
    # "void mb::attention::(anonymous namespace)::attention_wgmma_kernel<64, 0, false>(...)" -> "attention_wgmma_kernel"
    kernel = kernel.replace("(anonymous namespace)::", "")
    return kernel.split("(")[0].split("<")[0].split("::")[-1].split(" ")[-1]


def _calls(enc, vocab, rng):
    """(name, call) for every encode entry point of enc's towers; each call has a batch size of its own, so that its
    first use is the eager pass of a new CUDA-graph key."""
    calls, n = [], iter(range(1, 64))
    for normalize in (False, True):
        if enc.image_size:
            S = enc.image_size
            for name, shape in (("u8", (S, S)), ("u8 resized", (S + 37, S - 21))):
                img = rng.integers(0, 256, size=(next(n),) + shape + (3,), dtype=np.uint8)
                calls.append((f"{name} normalize={normalize}",
                              lambda img=img, nz=normalize: enc.encode_images_u8(img, nz)))
            chw = rng.standard_normal((next(n), 3, S, S)).astype(np.float32)
            calls.append((f"f32 normalize={normalize}", lambda chw=chw, nz=normalize: enc.encode_images_f32(chw, nz)))
        for masked in (False, True):
            b = next(n)
            ids = rng.integers(2, vocab - 1, size=(b, SEQ)).astype(np.int32)
            ids[:, -1] = vocab - 1
            lens = rng.integers(2, SEQ + 1, size=b)
            mask = (np.arange(SEQ)[None, :] < lens[:, None]).astype(np.int32) if masked else None
            calls.append((f"tokens mask={masked} normalize={normalize}",
                          lambda ids=ids, mk=mask, nz=normalize: enc.encode_tokens(ids, mk, nz)))
    return calls


@pytest.mark.parametrize("make", [_clip, _siglip, _clip_resnet, _clip_eva, _bert, _mpnet, _xlmr, _gte],
                         ids=["clip", "siglip", "clip_resnet", "clip_eva", "bert", "mpnet", "xlmr", "gte"])
def test_reported_launches_equal_the_kernels_run(gpu_required, make):
    from marqo_b200.engine import Encoder
    arch_name, arch, sd, vocab = make()
    enc = Encoder(arch_name, arch, sd, max_batch=64)
    torch.cuda.init()
    try:
        for name, call in _calls(enc, vocab, np.random.default_rng(0)):
            ran = _kernels(call)   # first use of the shape: eager
            eager = enc.last_timing()[1]
            assert eager > 0 and len(ran) == eager, f"{name}: reported {eager}, ran {len(ran)}: {ran}"
            call()                 # captured
            call()                 # replayed
            assert enc.last_timing()[1] == eager, f"{name}: graph replay"

            enc.set_profiling(True)
            try:
                base = [_base_name(k) for k in _kernels(call)]
                prof = enc.profile()
            finally:
                enc.set_profiling(False)
            assert prof["gemm_launches"] == sum(b.startswith("gemm") for b in base), f"{name}: {base}"
            assert prof["attention_launches"] == sum("attention" in b for b in base), f"{name}: {base}"
    finally:
        enc.close()


# Run in a process of its own: a torch.profiler session leaves CUPTI in a state in which a later session of the same
# process can miss the first kernels of a new model's stream.  argv[1]: [registry name, kind, arch edits, input].
_LAUNCHES_CHILD = """
import json, sys
import numpy as np, torch
from torch.profiler import ProfilerActivity, profile
from marqo_b200 import model_registry as R
from marqo_b200.engine import Encoder
from marqo_b200.weights import random_weights
name, kind, edits, (inp, shape) = json.loads(sys.argv[1])
arch = R.get_model_properties(name)["arch"]
for path, value in edits.items():
    *outer, key = path.split(".")
    d = arch
    for k in outer:
        d = d[k]
    d[key] = value
enc = Encoder(kind, arch, random_weights(kind, arch, 5), max_batch=shape[0])
rng = np.random.default_rng(5)
if inp == "u8":
    img = rng.integers(0, 256, tuple(shape) + (3,), dtype=np.uint8)
    run = lambda: enc.encode_images_u8(img)
else:   # token ids, row 3 masked after 100 tokens
    ids = rng.integers(103, 30000, tuple(shape)).astype(np.int32)
    mask = np.ones_like(ids)
    mask[3, 100:] = 0
    run = lambda: enc.encode_tokens(ids, mask)
run()   # warm-up
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    run()
    torch.cuda.synchronize()
ran = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
       and not e.name.startswith(("Memcpy", "Memset"))]
print(json.dumps({"reported": enc.last_timing()[1], "ran": ran}))
enc.close()
"""

_PHOTOS = ("u8", [4, 480, 640])
_EVA02 = {"rope_qk_kernel": 2, "swiglu_ln_kernel": 2, "attention_wgmma_kernel": 2}
# (registry name, kind, arch edits, input, reported launches, launches of named kernels)
_SERVED = {
    # the resize's two passes, embed rows, patch GEMM, 2 layers x (LN, QKV, rope, attention, attn.norm, out-proj, LN,
    # fc1, swiglu_ln, fc2), the head's LN, GEMM and L2
    "EVA02-B-16": ("open_clip/EVA02-B-16/merged2b_s8b_b131k", "clip_eva", {"layers": 0, "eva.layers": 2}, _PHOTOS,
                   2 + 2 + 2 * 10 + 3, _EVA02),
    "EVA02-L-14-336": ("open_clip/EVA02-L-14-336/merged2b_s6b_b61k", "clip_eva", {"layers": 0, "eva.layers": 2},
                       _PHOTOS, 2 + 2 + 2 * 10 + 3, _EVA02),
    # the resize's two passes, embed rows, patch GEMM, ln_pre, 2 layers x (LN, QKV, attention, out-proj, LN, fc1,
    # fc2), the head's 3
    "ViT-H-14-378": ("open_clip/ViT-H-14-378-quickgelu/dfn5b", "clip", {"text": None, "vision.layers": 2}, _PHOTOS,
                     2 + 3 + 2 * 7 + 3, {"attention_wgmma_kernel": 2}),
    "ViT-bigG-14": ("open_clip/ViT-bigG-14/laion2b_s39b_b160k", "clip", {"text": None, "vision.layers": 2}, _PHOTOS,
                    2 + 3 + 2 * 7 + 3, {"attention_wgmma_kernel": 2}),
    # stem GEMM + LN, 3 x (LN-patchify + GEMM), 5 blocks x 3, pool_ln, the MLP head's 2 GEMMs, l2
    "convnext_large_d": ("open_clip/convnext_large_d/laion2b_s26b_b102k_augreg", "clip_convnext",
                         {"layers": 0, "convnext.depths": [1, 1, 2, 1]}, ("u8", [4, 256, 256]),
                         2 + 3 * 2 + 5 * 3 + 1 + 2 + 1, {}),
    # embed, 2 layers x (QKV, rope, attention, o_proj, attn_ln, up_gate, geglu, down, mlp_ln), the head
    "Stella": ("Marqo/dunzhang-stella_en_400M_v5", "gte", {"layers": 2}, ("ids", [8, 300]), 1 + 2 * 9 + 1,
               {"rope_qk_kernel": 2, "geglu_kernel": 2, "bert_embed_ln_kernel": 1}),
}


@pytest.mark.parametrize("row", list(_SERVED))
def test_served_model_launches(gpu_required, row):
    """4 images (ConvNeXt at its own size, the others 480 x 640 through the resize) or 8 x 300 ids with one row
    masked, after a warm-up call."""
    name, kind, edits, inp, reported, kernels = _SERVED[row]
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([root, os.environ.get("PYTHONPATH", "")]))
    r = subprocess.run([sys.executable, "-c", _LAUNCHES_CHILD, json.dumps([name, kind, edits, inp])], cwd=root,
                       env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    assert out["reported"] == reported
    assert len(out["ran"]) == out["reported"], out["ran"]
    for kernel, n in kernels.items():
        assert sum(kernel in k for k in out["ran"]) == n, kernel
