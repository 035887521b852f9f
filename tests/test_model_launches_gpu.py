"""The launch count b200_model_last_timing reports, and the GEMM / attention launches b200_model_profile brackets, equal
the kernels the device ran (torch.profiler's CUDA kernel events) for one small model of every tower kind, through
every encode entry point, with and without L2 normalisation; and a replayed CUDA graph reports the count of the eager
pass it was captured from."""
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
