"""Every served transformer-layer variant through the shared layer runner (model.cu: run_layers), stage by stage,
against fp64.

Each kernel a layer launches has its own test through its own hook; this file checks their composition: which
buffers, widths, strides, scales, masks, tables and weights run_layers hands each kernel.  b200_debug_layers runs
layers [first, first + count) of a finalized model on residual rows the test owns and returns what the last layer left
in qkv (after any rotary embedding), o (the attention output), h (the last LayerNorm output), u (after the
activation or gate) and x.  Each stage is compared with fp64 arithmetic on the bf16-rounded weights, fed with the
engine's own previous stage, so a stage's bound depends on that stage only:

  a. qkv = bf16(LN1(x_in)) W_qkv^T + b (post-LN: bf16(x_in)), then the rotary embedding with fp64 angles;
  b. o = attention of the engine's qkv under the tower's mask and key lengths, MPNet's relative bias, scale
     1 / sqrt(the model's head dim), within test_attention_exact_gpu._bound; pad columns exactly 0;
  c. h = bf16(LN2(x_mid)) and u = act(h W_fc^T + b), x_mid = x_in + o' W_o^T + b_o (o' = bf16(attn.norm(o)) for EVA02; post-LN:
     x_mid = LN1(...)), or the gate (SwiGLU with its LayerNorm over the true hidden size, GeGLU); pad columns 0;
  d. x_out = x_mid + u W_proj^T + b (post-LN: LN2 of it).

Stages a, c and d carry an interval through the engine's own arithmetic: a centre (the fp64 value of the engine's
formula, with every bf16 rounding the engine stores applied to the centre) and a radius that bounds the distance of
the engine's value from it, per element.  Each step's radius is derived where the step is (see _linear, _layernorm,
_rounded and the activations), from the kernels' documented arithmetic; the checks are per element, and the worst
error / radius ratio of each stage is printed.

Stage c is split where the engine's own value is visible.  A pre-LN layer leaves fc1's input, bf16(LN2(x_mid)), in
h.  h is checked against its interval, and u is computed from the engine's h.  Otherwise the worst-case radius of
x_mid (the tensor core's K 2^-23 term) would make most LN2 outputs straddle a bf16 rounding boundary, and the ulp each
one carries, summed through |W_fc|, would hide an activation, LN2 or fc1 error of several percent.  A post-LN layer's
last LayerNorm overwrites h with bf16(x_out), which stage d checks bit for bit.  There u still starts from the interval
bf16(x_mid), so its bound is the wider one.

Bit-level checks: layers [0, 2) equal [0, 1) followed by [1, 2), and sequence 1 of a batch of 3 equals its run alone.

The cases are built from model_registry.served_models(): one per distinct layer variant (test_served_layer_variants
pins the set), with seeded weights from marqo_b200.weights at 2 layers, so that layer 1 alone makes the layer index
matter.  Text towers with key lengths run ragged lengths including 1 and S, at S below and above 128 (both attention
kernels).  For each width with a GEMM the persistent kernel can run (K >= 1024, N % 256 == 0), one case adds a batch
with at least one wave of its 128 x 256 tiles."""
import math
import zlib

import numpy as np
import pytest
import torch

import _gte_oracle as G
from marqo_b200 import _native as N
from marqo_b200 import model_registry as R
from marqo_b200 import weights as Wt
from test_attention_exact_gpu import CAUSAL, KEYLEN, MASK_NAME, NONE, _assert_bits, _nkb, _within_bound
from test_big_vit_kernels_gpu import _keep
from test_eva02_kernels_gpu import _theta

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available(), reason="needs an H100 (sm_90a)")]

LAYERS = 2
VOCAB = 64             # the layers never read the token table: a small one keeps the models quick to build
U = 2.0 ** -24         # fp32 unit roundoff
LOG2E = math.log2(math.e)
SHORT_S, LONG_S = 77, 257   # key-length towers: the mma.sync kernel (S < 128) and the wgmma one


# ------------------------------------------------------------------------------------------------------------ cases
def _kernel_hd(hd):
    return hd if hd <= 64 else 96 if hd <= 96 else 128      # model.cu: kernel_head_dim


def _case(out, key, **kw):
    cid = "-".join(str(k) for k in key)
    out.setdefault(cid, dict(id=cid, **kw))


def _variants():
    """{id: case} for every distinct transformer-layer variant the registry serves."""
    out = {}
    for _, e in sorted(R.served_models().items()):
        a = e["arch"]
        kind = a.get("kind", "clip" if "vision" in a else "bert")
        if kind == "clip":
            v, t = a["vision"], a["text"]
            S = (v["image_size"] // v["patch"]) ** 2 + 1
            _case(out, ("clip-vision", v["width"], v["mlp"], a["act"], S), fam="clip", kind="clip", tower="vision",
                  w=v["width"], heads=v["heads"], mlp=v["mlp"], act=a["act"], eps=1e-5, S=S, mask=NONE,
                  arch={"embed_dim": a["embed_dim"], "act": a["act"], "mean": a["mean"], "std": a["std"],
                        "vision": dict(v, layers=LAYERS)})
        if kind in ("clip", "clip_resnet", "clip_convnext", "clip_eva"):
            t = a["text"] if kind == "clip" else {k: a[k] for k in ("width", "heads", "mlp", "ctx")}
            _case(out, ("clip-text", t["width"], t["mlp"], a["act"], t["ctx"]), fam="clip", kind="clip", tower="text",
                  w=t["width"], heads=t["heads"], mlp=t["mlp"], act=a["act"], eps=1e-5, S=t["ctx"], mask=CAUSAL,
                  arch={"embed_dim": a["embed_dim"], "act": a["act"],
                        "text": dict(t, layers=LAYERS, vocab=VOCAB)})
        if kind == "clip_eva":
            ev = a["eva"]
            S = (ev["image_size"] // ev["patch"]) ** 2 + 1
            _case(out, ("eva-vision", ev["width"], ev["mlp"], S), fam="eva", kind="clip_eva", tower="vision",
                  w=ev["width"], heads=ev["heads"], mlp=ev["mlp"], act="swiglu", eps=ev["ln_eps"], S=S, mask=NONE,
                  grid=ev["image_size"] // ev["patch"], ref_grid=ev["rope_ref_grid"],
                  arch=dict(a, layers=0, eva=dict(ev, layers=LAYERS)))
        if kind == "siglip":
            v, t = a["vision"], a["text"]
            S = (v["image_size"] // v["patch"]) ** 2
            base = {k: a[k] for k in ("embed_dim", "act", "mean", "std", "ln_eps")}
            _case(out, ("siglip-vision", v["width"], v["mlp"], S), fam="timm", kind="siglip", tower="vision",
                  w=v["width"], heads=v["heads"], mlp=v["mlp"], act=a["act"], eps=a["ln_eps"], S=S, mask=NONE,
                  arch=dict(base, vision=dict(v, layers=LAYERS)))
            _case(out, ("siglip-text", t["width"], t["mlp"], t["ctx"]), fam="clip", kind="siglip", tower="text",
                  w=t["width"], heads=t["heads"], mlp=t["mlp"], act=a["act"], eps=a["ln_eps"], S=t["ctx"], mask=NONE,
                  arch=dict(base, text=dict(t, layers=LAYERS, vocab=VOCAB)))
        if kind in ("bert", "xlmr", "mpnet", "gte"):
            eps = 1e-12 if kind == "bert" else a["ln_eps"]
            # the text tower's token limit (engine.Encoder): RoBERTa positions start after the pad id
            tokens = {"gte": lambda: a["ctx"], "bert": lambda: a["max_pos"]}.get(
                kind, lambda: a["max_pos"] - a["pad_id"] - 1)()
            _case(out, (kind, a["width"], a["mlp"]), fam=kind, kind=kind, tower="text", w=a["width"],
                  heads=a["heads"], mlp=a["mlp"], act="geglu" if kind == "gte" else "gelu", eps=eps, S=tokens,
                  mask=KEYLEN, arch=dict(a, layers=LAYERS, vocab=VOCAB))
    for c in out.values():
        hd = c["w"] // c["heads"]
        c["hd"], c["aw"] = hd, c["heads"] * _kernel_hd(hd)
        gated = c["act"] in ("swiglu", "geglu")
        c["hp"] = -(-c["mlp"] // 64) * 64
        c["fc1"] = 2 * c["hp"] if gated else c["mlp"]
        c["pre_ln"] = c["fam"] in ("clip", "timm", "eva")
    # one case per width whose layer has a GEMM the persistent kernel can take gets a batch of at least one wave
    waved = set()
    for cid in sorted(out):
        c = out[cid]
        c["wave"] = bool(_persistent_gemms(c)) and c["w"] not in waved
        if c["wave"]:
            waved.add(c["w"])
    return out


def _persistent_gemms(c):
    """(N, K) of the layer's GEMMs the persistent kernel runs once M is large enough (gemm.cuh: K >= 1024, N % 256 == 0)."""
    gemms = [(3 * c["aw"], c["w"]), (c["w"], c["aw"]), (c["fc1"], c["w"]), (c["w"], c["fc1"] // 2 if
                                                                             c["act"] in ("swiglu", "geglu") else c["mlp"])]
    return [(n, k) for n, k in gemms if k >= 1024 and n % 256 == 0]


def _wave_rows(c, sms):
    """The fewest rows that give one of the layer's persistent-eligible GEMMs at least sms 128 x 256 tiles."""
    return min(128 * (-(-sms // (n // 256)) - 1) + 1 for n, _ in _persistent_gemms(c))


VARIANTS = _variants()


def test_served_layer_variants():
    """The enumeration reaches every layer variant the registry serves today: a table it stops reaching shows here."""
    v = VARIANTS.values()
    vit = {(c["w"], c["hd"], c["act"]) for c in v if c["fam"] == "clip" and c["tower"] == "vision"}
    assert {(768, 64, "gelu"), (768, 64, "quickgelu"), (1024, 64, "gelu"), (1024, 64, "quickgelu"), (1280, 80, "gelu"),
            (1408, 88, "gelu"), (1664, 104, "gelu")} <= vit
    assert {c["S"] for c in v if c["fam"] == "clip" and c["tower"] == "vision"} >= {50, 197, 257, 730}
    assert {c["w"] for c in v if c["fam"] == "clip" and c["tower"] == "text" and c["mask"] == CAUSAL} >= {
        512, 640, 768, 1024, 1280}
    assert {c["S"] for c in v if c["fam"] == "timm"} >= {196, 256, 576, 1024}
    assert {(c["S"], c["mask"]) for c in v if c["kind"] == "siglip" and c["tower"] == "text"} == {(64, NONE)}
    assert {c["w"] for c in v if c["kind"] == "bert"} >= {384, 768, 1024}
    assert {c["kind"] for c in v if c["mask"] == KEYLEN} == {"bert", "mpnet", "xlmr", "gte"}
    assert {(c["w"], c["mlp"], c["hp"], c["S"]) for c in v if c["fam"] == "eva"} >= {
        (768, 2048, 2048, 197), (1024, 2730, 2752, 257), (1024, 2730, 2752, 577)}
    assert any(c["fam"] == "gte" and c["fc1"] == 2 * c["mlp"] for c in v)
    widths = {c["w"] for c in v if _persistent_gemms(c)}
    assert widths >= {512, 768, 1024, 1280, 1408, 1664}
    assert {c["w"] for c in v if c["wave"]} == widths


# ---------------------------------------------------------------------------------------------------- the models
@pytest.fixture(scope="module")
def sm_count(gpu_required):
    return torch.cuda.get_device_properties(0).multi_processor_count


def _shapes(c, sms):
    """(B, S, key lengths) of the stage runs."""
    S = c["S"]
    if c["mask"] != KEYLEN:
        shapes = [(2, S, None)]
        if c["wave"]:
            shapes.append((-(-_wave_rows(c, sms) // S), S, None))
        return shapes
    shapes = [(4, SHORT_S, [SHORT_S, 1, 64, 40]), (4, LONG_S, [LONG_S, 1, 129, 64])]
    if c["wave"]:
        B = -(-_wave_rows(c, sms) // LONG_S)
        lens = torch.randint(1, LONG_S + 1, (B,), generator=torch.Generator().manual_seed(B)).tolist()
        shapes.append((B, LONG_S, [LONG_S, 1] + lens[2:]))
    return shapes


@pytest.fixture(scope="module", params=sorted(VARIANTS), ids=str)
def layer_model(request, sm_count):
    """(case, encoder, state dict) of one variant; module scope, so pytest runs a variant's tests together."""
    from marqo_b200.engine import Encoder
    c = VARIANTS[request.param]
    seed = zlib.crc32(c["id"].encode())
    sd = Wt.random_weights(c["kind"], c["arch"], seed)
    max_batch = max(max(b for b, _, _ in _shapes(c, sm_count)), 4)
    enc = Encoder(c["kind"], c["arch"], sd, max_batch=max_batch)
    from marqo_b200.engine import layer_cols
    # the library's buffer widths are the ones this file expects (model.cu: kernel_head_dim, fc1_cols)
    assert layer_cols(enc, c["tower"]) == (c["w"], c["aw"], c["fc1"])
    yield c, enc, sd
    enc.close()


# ------------------------------------------------------------------------------------------ fp64 interval steps
def _rnd(v):
    """fp64 -> fp32 -> bf16, back to fp64: monotone, and exactly the engine's rounding of an fp32 value."""
    return v.float().bfloat16().double()


def _rounded(c, r):
    """An fp32 value within r of c, rounded to bf16 (round to nearest even, as every bf16 store of the engine): the
    rounding is monotone, so the result lies in [rnd(c - r), rnd(c + r)]; the new centre is rnd(c) and the radius the
    larger distance of those ends from it (0 where both round alike).  2^-40 |c| covers the fp64 arithmetic of c -+ r."""
    r = r + 2.0 ** -40 * c.abs()
    rc = _rnd(c)
    return rc, torch.maximum(rc - _rnd(c - r), _rnd(c + r) - rc)


def _linear(a, ar, W, b, K, res=None, res_r=None):
    """The wgmma GEMM over bf16 rows within ar of a: a W^T + b (+ res), fp32 out.  Radius: ar through |W|; the tensor
    core's fp32 sum, exact products with one truncation per group of four (the bound test_attention_exact_gpu._bound
    uses: K 2^-23 of sum |a_k W_jk|, K the GEMM's depth with any zero padding); the epilogue's fp32 bias and residual
    additions (2^-23 of the magnitudes); and the residual's own radius."""
    c = a @ W.t()
    mag = (a.abs() + ar) @ W.abs().t()
    r = K * 2.0 ** -23 * mag + 2.0 ** -23 * c.abs()
    if bool((ar > 0).any()):
        r = r + ar @ W.abs().t()
    if b is not None:
        c = c + b
        r = r + 2.0 ** -23 * b.abs()
    if res is not None:
        c = c + res
        r = r + 2.0 ** -23 * (c.abs() + res.abs()) + (0 if res_r is None else res_r)
    return c, r


def _layernorm(x, xr, g, b, eps):
    """kernels.cu ln_row over rows within xr of x (fp32 in, fp32 out): centre, the fp64 LayerNorm of x.  Radius:
    (1) the input radius through the LayerNorm's Jacobian, d y_k / d x_j = g_k rstd (delta_kj - 1/w - xh_k xh_j / w),
    to first order |g_k| rstd (xr_k + mean xr + |xh_k| mean(|xh| xr)); (2) the kernel's fp32 arithmetic: the mean and
    the sum of squares each take n = w / 32 + 8 sequential additions per row (w / 128 float4 loads of four per lane,
    five shuffle levels), so |d mean| <= n 2^-24 mean |x| and rstd is off by at most (n + 8) 2^-24 relatively (the sum,
    the division by w, + eps, sqrtf, the reciprocal); y = (x - mean) rstd g + b adds four roundings of 2^-24.  Both
    are doubled to cover the second-order terms and the input rows' own magnitudes (|x| <= |x_c| + xr)."""
    w = x.shape[-1]
    mu = x.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((x - mu) ** 2).mean(-1, keepdim=True) + eps)
    xh = (x - mu) * rstd
    y = xh * g + b
    n = w / 32 + 8
    prop = g.abs() * rstd * (xr + xr.mean(-1, keepdim=True) + xh.abs() * (xh.abs() * xr).mean(-1, keepdim=True))
    own = U * (n * g.abs() * rstd * (x.abs() + xr).mean(-1, keepdim=True) + (n + 8) * g.abs() * xh.abs()
               + 4 * (y.abs() + b.abs()))
    return y, 2 * (prop + own)


def _gelu(z):
    return 0.5 * z * (1.0 + torch.erf(z / math.sqrt(2.0)))


def _act(z, zr, act):
    """fc1's epilogue activation over fp32 values within zr of z, before its bf16 store.  Both activations have a
    derivative of at most 1.13 (erf-GELU's largest, at z = sqrt 2).  The evaluation errors are the ones gemm.cu keeps
    (tests/test_gemm_shapes_gpu._edge_bound without its bf16 rounding): bf16-out erf-GELU runs in fp16, 2^-9 |z| +
    2^-24; QuickGELU (2^-21 + 2^-22 1.702 log2(e) |z|) |ref| + 2^-126 (1 + |z|)."""
    za = z.abs() + zr
    if act == "quickgelu":
        ref = z * torch.sigmoid(1.702 * z)
        err = (2.0 ** -21 + 2.0 ** -22 * 1.702 * LOG2E * za) * (ref.abs() + 1.13 * zr) + 2.0 ** -126 * (1 + za)
    else:
        ref = _gelu(z)
        err = 2.0 ** -9 * za + 2.0 ** -24
    return ref, 1.13 * zr + err


def _check(stage, got, c, r):
    """Every element of got within r of c (exactly c where r is 0) -> the worst ratio |got - c| / r."""
    err = (got - c).abs()
    over = err > r
    if bool(over.any()):
        i = tuple(over.nonzero()[0].tolist())
        pytest.fail(f"{stage}: {int(over.sum())} of {over.numel()} elements over the bound, first at {i}: got "
                    f"{float(got[i])!r}, ref {float(c[i])!r}, bound {float(r[i]):.3g}")
    live = r > 0
    return float((err[live] / r[live]).max()) if bool(live.any()) else 0.0


# ------------------------------------------------------------------------------------------------- layer weights
def _layer(c, sd, i):
    """Layer i's parameters in the checkpoint's own (unpadded) layout, on the GPU in fp64: Linear weights rounded to
    bf16 as the engine stores them, biases and LayerNorms as uploaded (fp32)."""
    def f(name):
        return torch.from_numpy(np.asarray(sd[name], np.float32)).cuda().double()

    def lin(name):
        return torch.from_numpy(np.asarray(sd[name], np.float32)).cuda().bfloat16().double()

    w, fam = c["w"], c["fam"]
    zeros = torch.zeros(w, dtype=torch.float64, device="cuda")
    L = {}
    if fam == "clip":
        p = {"vision": "visual.", "text": "text." if c["kind"] == "siglip" else ""}[c["tower"]]
        p = f"{p}transformer.resblocks.{i}."
        L.update(ln1=(f(p + "ln_1.weight"), f(p + "ln_1.bias")), ln2=(f(p + "ln_2.weight"), f(p + "ln_2.bias")),
                 wqkv=lin(p + "attn.in_proj_weight"), bqkv=f(p + "attn.in_proj_bias"),
                 wo=lin(p + "attn.out_proj.weight"), bo=f(p + "attn.out_proj.bias"),
                 wfc=lin(p + "mlp.c_fc.weight"), bfc=f(p + "mlp.c_fc.bias"),
                 wproj=lin(p + "mlp.c_proj.weight"), bproj=f(p + "mlp.c_proj.bias"))
    elif fam == "timm":
        p = f"visual.trunk.blocks.{i}."
        L.update(ln1=(f(p + "norm1.weight"), f(p + "norm1.bias")), ln2=(f(p + "norm2.weight"), f(p + "norm2.bias")),
                 wqkv=lin(p + "attn.qkv.weight"), bqkv=f(p + "attn.qkv.bias"),
                 wo=lin(p + "attn.proj.weight"), bo=f(p + "attn.proj.bias"),
                 wfc=lin(p + "mlp.fc1.weight"), bfc=f(p + "mlp.fc1.bias"),
                 wproj=lin(p + "mlp.fc2.weight"), bproj=f(p + "mlp.fc2.bias"))
    elif fam == "eva":
        p = f"visual.trunk.blocks.{i}."
        a = p + "attn."
        L.update(ln1=(f(p + "norm1.weight"), f(p + "norm1.bias")), ln2=(f(p + "norm2.weight"), f(p + "norm2.bias")),
                 wqkv=torch.cat([lin(a + "q_proj.weight"), lin(a + "k_proj.weight"), lin(a + "v_proj.weight")]),
                 bqkv=torch.cat([f(a + "q_proj.bias"), zeros, f(a + "v_proj.bias")]),   # k_proj has no bias
                 ln_attn=(f(a + "norm.weight"), f(a + "norm.bias")),
                 wo=lin(a + "proj.weight"), bo=f(a + "proj.bias"),
                 wg=lin(p + "mlp.fc1_g.weight"), bg=f(p + "mlp.fc1_g.bias"),
                 wx=lin(p + "mlp.fc1_x.weight"), bx=f(p + "mlp.fc1_x.bias"),
                 ln_mlp=(f(p + "mlp.norm.weight"), f(p + "mlp.norm.bias")),
                 wproj=lin(p + "mlp.fc2.weight"), bproj=f(p + "mlp.fc2.bias"))
    elif fam in ("bert", "xlmr", "mpnet"):
        p = f"encoder.layer.{i}."
        if fam == "mpnet":
            q, o, ln1 = p + "attention.attn.", p + "attention.attn.o.", p + "attention.LayerNorm."
            parts = ("q", "k", "v")
        else:
            q, o, ln1 = p + "attention.self.", p + "attention.output.dense.", p + "attention.output.LayerNorm."
            parts = ("query", "key", "value")
        L.update(ln1=(f(ln1 + "weight"), f(ln1 + "bias")),
                 ln2=(f(p + "output.LayerNorm.weight"), f(p + "output.LayerNorm.bias")),
                 wqkv=torch.cat([lin(f"{q}{n}.weight") for n in parts]),
                 bqkv=torch.cat([f(f"{q}{n}.bias") for n in parts]),
                 wo=lin(o + "weight"), bo=f(o + "bias"),
                 wfc=lin(p + "intermediate.dense.weight"), bfc=f(p + "intermediate.dense.bias"),
                 wproj=lin(p + "output.dense.weight"), bproj=f(p + "output.dense.bias"))
    else:   # gte: up_gate_proj is up | gate, without a bias
        p = f"encoder.layer.{i}."
        ug = lin(p + "mlp.up_gate_proj.weight")
        L.update(ln1=(f(p + "attn_ln.weight"), f(p + "attn_ln.bias")), ln2=(f(p + "mlp_ln.weight"), f(p + "mlp_ln.bias")),
                 wqkv=lin(p + "attention.qkv_proj.weight"), bqkv=f(p + "attention.qkv_proj.bias"),
                 wo=lin(p + "attention.o_proj.weight"), bo=f(p + "attention.o_proj.bias"),
                 wup=ug[:c["mlp"]], wgate=ug[c["mlp"]:],
                 wproj=lin(p + "mlp.down_proj.weight"), bproj=f(p + "mlp.down_proj.bias"))
    return L


def _rope_angles(c, S):
    """[S, 32] fp64 angles of each token row of a sequence, or None (no rotary embedding).  EVA02: the class row has
    none (its rows are those of the patches after it); GTE: position s from row 0."""
    if c["fam"] == "eva":
        return _theta(c["grid"], c["ref_grid"]).cuda()
    if c["fam"] == "gte":
        a = c["arch"]
        return G.rope_angles(G.GteCfg(rope_theta=a["rope_theta"], rope_ntk_factor=a["rope_ntk_factor"]), S).cuda()
    return None


def _rel_bias_log2(c, sd, S):
    """MPNet's relative-position bias in log2 units, [1, H, S, S]: bias[h, i, j] = weight[bucket(j - i), h]."""
    if c["fam"] != "mpnet":
        return None
    from marqo_b200.engine import relative_position_buckets
    a = c["arch"]
    bucket = torch.from_numpy(relative_position_buckets(S, a["rel_buckets"], a["rel_max_distance"])).long().cuda()
    wt = torch.from_numpy(np.asarray(sd["encoder.relative_attention_bias.weight"], np.float32)).cuda().double()
    key = torch.arange(S, device="cuda")
    table = wt[bucket[key[None, :] - key[:, None] + S - 1]]          # [S, S, H]
    return table.permute(2, 0, 1)[None] * LOG2E


# ---------------------------------------------------------------------------------------------------- the stages
def _stage_a(c, L, x, B, S, got_qkv):
    """qkv of rows x -> worst ratio.  Pre-LN: bf16(LN1(x)); post-LN: bf16(x), exactly what the hook leaves in h."""
    w, H, hd, hdp = c["w"], c["heads"], c["hd"], c["aw"] // c["heads"]
    if c["pre_ln"]:
        h, hr = _rounded(*_layernorm(x, torch.zeros_like(x), *L["ln1"], c["eps"]))
    else:
        h, hr = _rnd(x), torch.zeros_like(x)
    z, zr = _rounded(*_linear(h, hr, L["wqkv"], L["bqkv"], w))
    th = _rope_angles(c, S)
    if th is not None:
        qk, qkr = z.view(B, S, 3, H, hd)[:, :, :2], zr.view(B, S, 3, H, hd)[:, :, :2]
        if c["fam"] == "eva":   # interleaved pairs (2j, 2j + 1), rows after the class row
            first, split = 1, lambda t: (t[..., 0::2], t[..., 1::2])
            ang = th[None, :, None, None, :]
        else:                   # rotate-half pairs (j, j + 32) from row 0
            first, split = 0, lambda t: (t[..., :32], t[..., 32:])
            ang = th[None, :S, None, None, :]
        cos, sin = ang.cos(), ang.sin()
        a_, b_ = split(qk[:, first:])
        ar, br = split(qkr[:, first:])
        # rope_qk: fp32 arithmetic on the table's fp32 (cos, sin), 2^-20 (|a| + |b|) (the rope_qk kernel tests), then
        # a second bf16 store
        mag = 2.0 ** -20 * (a_.abs() + ar + b_.abs() + br)
        na, nar = _rounded(a_ * cos - b_ * sin, cos.abs() * ar + sin.abs() * br + mag)
        nb, nbr = _rounded(b_ * cos + a_ * sin, cos.abs() * br + sin.abs() * ar + mag)
        z, zr = z.clone().view(B, S, 3, H, hd), zr.clone().view(B, S, 3, H, hd)
        for t, (ta, tb) in ((z, (na, nb)), (zr, (nar, nbr))):
            ca, cb = split(t[:, first:, :2])   # views into t
            ca.copy_(ta)
            cb.copy_(tb)
    got = got_qkv.double().view(B, S, 3, H, hdp)
    _assert_bits(got[..., hd:], torch.zeros_like(got[..., hd:]), "qkv pad columns")
    return _check("qkv", got[..., :hd], z.view(B, S, 3, H, hd), zr.view(B, S, 3, H, hd))


def _stage_b(c, sd, B, S, lens, got_qkv, got_o):
    """Attention of the engine's own qkv -> worst ratio (test_attention_exact_gpu._within_bound)."""
    H, hd, hdp = c["heads"], c["hd"], c["aw"] // c["heads"]
    o = got_o.view(B, S, H, hdp)
    _assert_bits(o[..., hd:], torch.zeros_like(o[..., hd:]), "o pad columns")
    q, k, v = got_qkv.view(B, S, 3, H, hdp)[..., :hd].double().permute(2, 0, 3, 1, 4)
    lens = lens or [S] * B
    return _within_bound(o[..., :hd].permute(0, 2, 1, 3).double(), q, k, v, _keep(B, S, c["mask"], lens),
                         _rel_bias_log2(c, sd, S), hdp, LOG2E / math.sqrt(hd), _nkb(S, c["mask"], lens), S, True)


def _stage_c(c, L, x, got_o, got_h, got_u):
    """h and u from the engine's o -> (worst ratio of h or None, worst ratio of u, the x_mid interval stage d starts
    from).  A pre-LN layer leaves fc1's input in h: it is checked against bf16(LN2(x_mid)), and u is then computed
    from the engine's own h, so u's bound holds only fc1's and the activation's arithmetic.  A post-LN layer's h is
    overwritten by its last LayerNorm (stage d), so its fc1 input is the interval bf16(x_mid)."""
    w, H, hd, hdp, K_o = c["w"], c["heads"], c["hd"], c["aw"] // c["heads"], c["aw"]
    o = got_o.double().view(-1, H, hdp)[..., :hd].reshape(-1, w)
    zero = torch.zeros_like(x)
    if "ln_attn" in L:   # EVA02's attn.norm over the bf16 attention output, stored bf16
        o, orr = _rounded(*_layernorm(o, torch.zeros_like(o), *L["ln_attn"], c["eps"]))
        K_o = w
    else:
        orr = torch.zeros_like(o)
    xm, xmr = _linear(o, orr, L["wo"], L["bo"], K_o, res=x, res_r=zero)
    ratio_h = None
    if c["pre_ln"]:
        ratio_h = _check("h", got_h.double(), *_rounded(*_layernorm(xm, xmr, *L["ln2"], c["eps"])))
        h2 = got_h.double()
        h2r = torch.zeros_like(h2)
    else:
        xm, xmr = _layernorm(xm, xmr, *L["ln1"], c["eps"])
        h2, h2r = _rounded(xm, xmr)
    got = got_u.double()
    mlp, hp = c["mlp"], c["hp"]
    if c["act"] == "swiglu":
        g, gr = _rounded(*_linear(h2, h2r, L["wg"], L["bg"], w))
        xx, xxr = _rounded(*_linear(h2, h2r, L["wx"], L["bx"], w))
        sg = g * torch.sigmoid(g)
        # silu(g) x in fp32 (__expf and three roundings, 2^-20 |g x|); silu' <= 1.1
        s = sg * xx
        sr = sg.abs() * xxr + 1.1 * gr * (xx.abs() + xxr) + 2.0 ** -20 * (g.abs() + gr) * (xx.abs() + xxr)
        u, ur = _rounded(*_layernorm(s, sr, *L["ln_mlp"], c["eps"]))
        ratio = max(_check("u", got[:, :mlp], u, ur), _check("u (fc1_x half)", got[:, hp:hp + mlp], xx, xxr))
        _assert_bits(got_u[:, mlp:hp], torch.zeros_like(got_u[:, mlp:hp]), "u pad columns")
        _assert_bits(got_u[:, hp + mlp:], torch.zeros_like(got_u[:, hp + mlp:]), "fc1_x pad columns")
    elif c["act"] == "geglu":
        up, upr = _rounded(*_linear(h2, h2r, L["wup"], None, w))
        gt, gtr = _rounded(*_linear(h2, h2r, L["wgate"], None, w))
        ge = _gelu(gt)
        # GELU_erf(gate) up in fp32: erff's 2 ulp and the roundings, 1e-6 |gate up| (test_gte_kernels_gpu)
        u, ur = _rounded(ge * up, ge.abs() * upr + 1.13 * gtr * (up.abs() + upr)
                         + 1e-6 * (gt.abs() + gtr) * (up.abs() + upr))
        ratio = max(_check("u", got[:, :mlp], u, ur), _check("u (gate half)", got[:, mlp:], gt, gtr))
    else:
        u, ur = _rounded(*_act(*_linear(h2, h2r, L["wfc"], L["bfc"], w), c["act"]))
        ratio = _check("u", got, u, ur)
    return ratio_h, ratio, (xm, xmr)


def _stage_d(c, L, xmid, got_u, got_x, got_h):
    """x_out from the engine's u and stage c's x_mid -> worst ratio.  A post-LN layer's last LayerNorm also leaves
    h = bf16(x_out), bit for bit."""
    xm, xmr = xmid
    mlp = c["mlp"]
    K = c["hp"] if c["act"] in ("swiglu", "geglu") else mlp
    z, zr = _linear(got_u[:, :mlp].double(), torch.zeros_like(xm[:, :1]).expand(-1, mlp), L["wproj"], L["bproj"],
                    K, res=xm, res_r=xmr)
    if not c["pre_ln"]:
        z, zr = _layernorm(z, zr, *L["ln2"], c["eps"])
        _assert_bits(got_h, got_x.bfloat16(), "h vs bf16(x) after the post-LN LayerNorm")
    return _check("x", got_x.double(), z, zr)


def _inputs(c, B, S, seed):
    """Residual rows [B * S, w]: unit Gaussians with a per-column offset, as a residual stream carries."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B * S, c["w"], generator=g, device="cuda")
    return x + 0.5 * torch.randn(1, c["w"], generator=g, device="cuda")


def _run(enc, c, first, count, x, S, lens):
    from marqo_b200.engine import debug_layers
    return debug_layers(enc, c["tower"], first, count, x, S, lens)


# ------------------------------------------------------------------------------------------------------ the tests
def test_layer_stages_within_bound(layer_model, sm_count):
    """Layer 0 from x_in, then layer 1 alone from layer 0's output: every stage of each within its fp64 bound."""
    c, enc, sd = layer_model
    for B, S, lens in _shapes(c, sm_count):
        x = _inputs(c, B, S, seed=B * 1000 + S)
        for i in range(LAYERS):
            out = _run(enc, c, i, 1, x, S, lens)
            L = _layer(c, sd, i)
            xd = x.double()
            ra = _stage_a(c, L, xd, B, S, out["qkv"])
            rb = _stage_b(c, sd, B, S, lens, out["qkv"], out["o"])
            rh, rc, xmid = _stage_c(c, L, xd, out["o"], out["h"], out["u"])
            rd = _stage_d(c, L, xmid, out["u"], out["x"], out["h"])
            h = "-" if rh is None else f"{rh:.3f}"
            print(f"\n[layer stages] {c['id']} layer {i} B={B} S={S} {MASK_NAME[c['mask']]}: worst ratio qkv {ra:.3f} "
                  f"o {rb:.3f} h {h} u {rc:.3f} x {rd:.3f}")
            x = out["x"]


def test_layer_ranges_compose_bit_for_bit(layer_model):
    """Layers [0, 2) give bitwise [0, 1) followed by [1, 2), in every buffer the last layer leaves."""
    c, enc, _ = layer_model
    B, S, lens = 3, c["S"], None
    if c["mask"] == KEYLEN:
        S, lens = LONG_S, [LONG_S, 1, 100]
    x = _inputs(c, B, S, seed=7)
    both = _run(enc, c, 0, 2, x, S, lens)
    one = _run(enc, c, 0, 1, x, S, lens)
    two = _run(enc, c, 1, 1, one["x"], S, lens)
    for k in ("x", "h", "qkv", "o", "u"):
        got, want = both[k], two[k]
        if k == "x":
            got, want = got.view(torch.int32).view(torch.bfloat16), want.view(torch.int32).view(torch.bfloat16)
        _assert_bits(got, want, f"{k}: layers [0, 2) vs [0, 1) then [1, 2)")
    assert not torch.equal(one["x"], both["x"]), "layer 1 left the residual stream unchanged"


def test_sequence_alone_bit_for_bit(layer_model):
    """Sequence 1 of a batch of 3 gives bitwise its run alone, through both layers."""
    c, enc, _ = layer_model
    S = c["S"] if c["mask"] != KEYLEN else SHORT_S
    lens = [S, S // 2 + 1, 1] if c["mask"] == KEYLEN else None
    x = _inputs(c, 3, S, seed=11)
    batch = _run(enc, c, 0, LAYERS, x, S, lens)
    alone = _run(enc, c, 0, LAYERS, x[S:2 * S].contiguous(), S, None if lens is None else lens[1:2])
    for k in ("x", "h", "qkv", "o", "u"):
        got, want = batch[k][S:2 * S], alone[k]
        if k == "x":
            got, want = got.view(torch.int32).view(torch.bfloat16), want.view(torch.int32).view(torch.bfloat16)
        _assert_bits(got, want, f"{k}: sequence 1 of 3 vs alone")


def test_debug_layers_refuses_bad_arguments(gpu_required):
    """A tower the model lacks, a layer range outside the tower, more rows than the workspace holds, a vision S other
    than the tower's token count and a key length outside 0..S are B200_ERR_INVALID_ARG."""
    from marqo_b200.engine import Encoder, debug_layers
    bert = VARIANTS["bert-384-1536"]
    vit = VARIANTS["clip-vision-768-3072-gelu-50"]
    encs = []
    try:
        eb = Encoder("bert", bert["arch"], Wt.random_weights("bert", bert["arch"], 1), max_batch=2)
        ev = Encoder("clip", vit["arch"], Wt.random_weights("clip", vit["arch"], 2), max_batch=2)
        encs += [eb, ev]
        xb = torch.zeros(2 * 16, 384, device="cuda")
        xv = torch.zeros(50, 768, device="cuda")
        for enc, tower, first, count, x, S in [
                (eb, "vision", 0, 1, xb, 16),                          # BERT has no vision tower
                (ev, "text", 0, 1, xv, 50),                            # this CLIP has no text tower
                (eb, "text", 2, 1, xb, 16), (eb, "text", 1, 2, xb, 16),   # beyond the 2 layers
                (eb, "text", -1, 1, xb, 16), (eb, "text", 0, 0, xb, 16),
                (eb, "text", 0, 1, torch.zeros(3 * 16, 384, device="cuda"), 16),   # 3 sequences, max_batch 2
                (eb, "text", 0, 1, torch.zeros(513, 384, device="cuda"), 513),    # beyond the tower's 512 tokens
                (ev, "vision", 0, 1, torch.zeros(49, 768, device="cuda"), 49),    # not the 50 tokens of an image
                (ev, "vision", 0, 1, torch.zeros(3 * 50, 768, device="cuda"), 50)]:
            with pytest.raises(N.NativeError) as ei:
                debug_layers(enc, tower, first, count, x, S)
            assert ei.value.code == N.ERR_INVALID_ARG, (tower, first, count, tuple(x.shape), S)
        for lens in ([16, 17], [-1, 16]):
            with pytest.raises(N.NativeError) as ei:
                debug_layers(eb, "text", 0, 1, xb, 16, lens)
            assert ei.value.code == N.ERR_INVALID_ARG, lens
        # and the model still runs: the refusals touched nothing
        debug_layers(eb, "text", 0, 2, xb, 16)
    finally:
        for e in encs:
            e.close()
