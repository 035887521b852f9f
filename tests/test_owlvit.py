"""The OWL-ViT image reranker on the CPU: the fp32 oracle against transformers' OwlViTForObjectDetection, the engine's
box bias table, the checkpoint rename, the 16-token query tokenisation against HF's CLIP tokenizers, the OWL_VIT_MODELS
table, the ReRankerOwl factory's routing, and the served subclass's rerank against the reference's per-image loop."""
import json
import types

import numpy as np
import pytest
import torch

import _owlvit_oracle as O

transformers = pytest.importorskip("transformers")


def _arch(vw, vl, vh, patch, size, tw, tl=1, vocab=1000):
    return {"embed_dim": tw, "act": "quickgelu", "resize_mode": "squash", "owl_detect": True,
            "vision": {"width": vw, "layers": vl, "heads": vh, "mlp": 4 * vw, "patch": patch, "image_size": size},
            "text": {"width": tw, "layers": tl, "heads": tw // 64, "mlp": 4 * tw, "ctx": 16, "vocab": vocab}}


def _hf_model(arch):
    v, t = arch["vision"], arch["text"]
    cfg = transformers.OwlViTConfig(
        text_config={"hidden_size": t["width"], "num_hidden_layers": t["layers"], "num_attention_heads": t["heads"],
                     "intermediate_size": t["mlp"], "vocab_size": t["vocab"], "max_position_embeddings": 16},
        vision_config={"hidden_size": v["width"], "num_hidden_layers": v["layers"], "num_attention_heads": v["heads"],
                       "intermediate_size": v["mlp"], "patch_size": v["patch"], "image_size": v["image_size"]},
        projection_dim=arch["embed_dim"])
    return transformers.OwlViTForObjectDetection(cfg).eval()


def _load_hf(model, sd):
    """Our random weights (checkpoint names) into a transformers model, whatever it calls the pre-LayerNorm."""
    own = model.state_dict()
    fixed = {}
    for k, v in sd.items():
        if k not in own and "pre_layrnorm" in k:
            k = k.replace("pre_layrnorm", "pre_layernorm")
        fixed[k] = torch.from_numpy(np.asarray(v)).reshape(own[k].shape)
    missing, unexpected = model.load_state_dict(fixed, strict=False)
    assert not unexpected and all(k.endswith("position_ids") for k in missing), (missing, unexpected)


SMALL = {"tiny_p16": _arch(128, 2, 2, 16, 64, 128, 2), "tiny_p8": _arch(256, 1, 4, 8, 64, 128, 1)}
# the three checkpoints' shapes, one layer per tower
REAL = {"B32": _arch(768, 1, 12, 32, 768, 512), "B16": _arch(768, 1, 12, 16, 768, 512),
        "L14": _arch(1024, 1, 16, 14, 840, 768)}


@pytest.mark.parametrize("name", sorted(SMALL) + sorted(REAL))
def test_oracle_matches_transformers(name):
    from marqo_b200 import weights as W
    arch = {**SMALL, **REAL}[name]
    sd = W.random_owlvit_weights(arch, 7)
    model = _hf_model(arch)
    _load_hf(model, sd)
    S = arch["vision"]["image_size"]
    g = torch.Generator().manual_seed(3)
    pixels = torch.randn(2, 3, S, S, generator=g)
    ids = torch.zeros(16, dtype=torch.int64)
    ids[:5] = torch.tensor([arch["text"]["vocab"] - 2, 17, 300, 42, arch["text"]["vocab"] - 1])
    with torch.no_grad():
        q = ids[None].expand(2, 16)   # one query per image, as the processor repeats it
        out = model(input_ids=q, pixel_values=pixels, attention_mask=(q != 0).long())
    logits, boxes = O.detect(sd, pixels, ids, arch["vision"]["heads"], arch["text"]["heads"])
    np.testing.assert_allclose(logits.numpy(), out.logits[..., 0].numpy(), rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(boxes.numpy(), out.pred_boxes.numpy(), rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("G", [24, 48, 60])
def test_box_bias_matches_transformers(native_lib, G):
    from marqo_b200.engine import owl_box_bias
    cls = transformers.OwlViTForObjectDetection
    ns = types.SimpleNamespace(normalize_grid_corner_coordinates=cls.normalize_grid_corner_coordinates)
    want = cls.compute_box_bias(ns, G, G).numpy()
    np.testing.assert_allclose(O.box_bias(G).numpy(), want, rtol=0, atol=0)
    # fp64 rounded once, against transformers' fp32: log1p(-c + 1e-4) cancels in fp32 at the last row and column
    # (c = 1), where the two differ by up to 1.7e-4 (logits near 9.2); everywhere else they agree to 2 ulp
    got = owl_box_bias(G)
    np.testing.assert_allclose(got, want, rtol=0, atol=3e-4)
    inner = np.asarray(O.box_bias(G).numpy()[:, :2] < 9.0).all(axis=1)
    np.testing.assert_allclose(got[inner], want[inner], rtol=3e-7, atol=1e-6)


def test_rename_uses_every_tensor():
    from marqo_b200 import weights as W
    arch = SMALL["tiny_p16"]
    model = _hf_model(arch)
    sd = {k: v.numpy() for k, v in model.state_dict().items()}
    eng = W.owlvit_state_dict_to_engine(sd)
    clip = set(W.random_clip_weights(arch, 1)) - {"visual.proj"}
    heads = {k for k in sd if k.startswith(("layer_norm.", "class_head.", "box_head."))}
    assert set(eng) == clip | heads
    used = {k for k in sd if not k.endswith("position_ids")}
    assert used - set(W.OWLVIT_UNUSED) - heads   # tower tensors exist and all of them were mapped (no KeyError)
    p = "owlvit.vision_model.encoder.layers.1.self_attn."
    want = np.concatenate([sd[p + "q_proj.weight"], sd[p + "k_proj.weight"], sd[p + "v_proj.weight"]])
    np.testing.assert_array_equal(eng["visual.transformer.resblocks.1.attn.in_proj_weight"], want)
    want = np.concatenate([sd[p + "q_proj.bias"], sd[p + "k_proj.bias"], sd[p + "v_proj.bias"]])
    np.testing.assert_array_equal(eng["visual.transformer.resblocks.1.attn.in_proj_bias"], want)
    np.testing.assert_array_equal(eng["text_projection"], sd["owlvit.text_projection.weight"].T)
    with pytest.raises(KeyError):
        W.owlvit_state_dict_to_engine({**sd, "owlvit.vision_model.extra.weight": np.zeros(1, np.float32)})


# ---------------------------------------------------------------------------------------------------- tokenizer
CORPUS = ["a photo of a cat", "a photo of a dog", "the red car on the street", "two people walking", "hello world",
          "a bowl of fruit", "photo photos photograph"] * 3


@pytest.fixture(scope="module")
def toy_tokenizers(native_lib, tmp_path_factory):
    from marqo_b200.tokenizers import ClipBpeTokenizer
    from oracle import tokenizers as OT
    merges = OT.train_toy_merges(CORPUS, 300)
    ref = OT.SimpleTokenizerOracle(merges)
    d = tmp_path_factory.mktemp("clipvocab")
    vocab = dict(ref.encoder)
    vocab["<|startoftext|>"] = vocab.pop("<start_of_text>")
    vocab["<|endoftext|>"] = vocab.pop("<end_of_text>")
    (d / "vocab.json").write_text(json.dumps(vocab))
    (d / "merges.txt").write_text(merges)
    hf = []
    for cls in ("CLIPTokenizer", "CLIPTokenizerFast"):
        try:
            tok = getattr(transformers, cls)(str(d / "vocab.json"), str(d / "merges.txt"), pad_token="!")
        except Exception:  # noqa: BLE001
            continue
        hf.append(tok)
    if not hf:
        pytest.skip("no HF CLIP tokenizer can be built offline here")
    return ClipBpeTokenizer(merges.encode("utf-8"), context_length=16), hf


@pytest.mark.parametrize("query", ["a photo of a cat", "the red car", "two people walking on the street",
                                   "hello", "a bowl of fruit photo photos"])
def test_query_ids_match_hf_clip_tokenizer(toy_tokenizers, query):
    from marqo_b200.owl_reranker import query_ids
    mine, hf = toy_tokenizers
    got = query_ids(mine, query).tolist()
    for tok in hf:
        want = tok(query, padding="max_length", max_length=16)["input_ids"]
        assert got == want, type(tok).__name__


def test_long_query_refused(toy_tokenizers):
    from marqo_b200.owl_reranker import query_ids
    mine, _ = toy_tokenizers
    assert query_ids(mine, " ".join(["cat"] * 14)).shape == (16,)   # 14 + <start> + <end>: exactly 16
    with pytest.raises(ValueError):
        query_ids(mine, " ".join(["cat"] * 15))


# ---------------------------------------------------------------------------------------------------- registry
def test_owl_vit_table():
    from marqo_b200 import model_registry as R
    assert sorted(R.OWL_VIT_MODELS) == sorted([
        "google/owlvit-base-patch32", "google/owlvit-base-patch16", "google/owlvit-large-patch14",
        "owl/ViT-B/32", "owl/ViT-B/16", "owl/ViT-L/14"])
    shapes = {ck: (e["arch"]["vision"]["width"], e["arch"]["vision"]["layers"], e["arch"]["vision"]["patch"],
                   e["arch"]["vision"]["image_size"], e["arch"]["embed_dim"])
              for e in R.OWL_VIT_MODELS.values() for ck in [e["checkpoint"]]}
    assert shapes == {"google/owlvit-base-patch32": (768, 12, 32, 768, 512),
                      "google/owlvit-base-patch16": (768, 12, 16, 768, 512),
                      "google/owlvit-large-patch14": (1024, 24, 14, 840, 768)}
    assert R.OWL_VIT_MODELS["owl/ViT-L/14"]["checkpoint"] == "google/owlvit-large-patch14"
    for name in R.OWL_VIT_MODELS:
        assert name not in R.all_models()


class _Stand:
    def __init__(self, *args, **kwargs):
        self.args, self.kwargs = args, kwargs


class _Original(_Stand):
    pass


class _Served(_Stand):
    pass


def test_factory_routes_served_names():
    from marqo_b200.owl_reranker import make_owl_factory
    f = make_owl_factory(_Original, _Served)
    assert f.original is _Original
    assert isinstance(f(model_name="owl/ViT-B/32", device="cuda", image_size=(240, 240)), _Served)
    assert isinstance(f("google/owlvit-large-patch14", "cuda:1", (240, 240)), _Served)
    assert isinstance(f(model_name="owl/ViT-B/32", device="cpu", image_size=(240, 240)), _Original)
    assert isinstance(f(model_name="owl/ViT-H/14", device="cuda", image_size=(240, 240)), _Original)
    o = f(model_name="owl/ViT-B/16", device="cpu", image_size=(240, 240))
    assert o.kwargs == {"model_name": "owl/ViT-B/16", "device": "cpu", "image_size": (240, 240)}


# ---------------------------------------------------------------------------------------------------- rerank loop
# Stand-ins for what the served subclass inherits and calls: Marqo's ReRankerOwl surface (its model map, the
# formatted inputs, the image loader, the reranked-results step) and the reranking helpers of cross_encoders.
class _Columns:
    query, field_content, original_field_name, bbox, bbox_original = (
        "query", "field_content", "original_field_name", "bbox", "bbox_original")


class _Fields:
    hits, reranker_score, reranked_id = "hits", "_reranked_score", "_rerank_id"


def _helpers():
    import logging
    import pandas as pd

    def sort_boxes(boxes, scores, identifier):
        inds = scores.argsort(descending=True)
        return boxes[inds], scores[inds], [identifier[i] for i in inds]

    def rescale(box, from_size, to_size):
        fx, fy = to_size[0] / from_size[0], to_size[1] / from_size[1]
        x1, y1, x2, y2 = box
        return [x1 * fx, y1 * fy, x2 * fx, y2 * fy]

    return types.SimpleNamespace(
        ResultsFields=_Fields, Columns=_Columns, logger=logging.getLogger("owl-test"), pd=pd,
        _process_owl_result=lambda r, ident: (r[0]["boxes"], r[0]["scores"], [ident] * len(r[0]["scores"])),
        sort_owl_boxes_scores=sort_boxes, _keep_top_k=lambda x, k=1: x[:k],
        image_processor=types.SimpleNamespace(rescale_box=rescale))


def _images(n, seed):
    from PIL import Image
    rng = np.random.default_rng(seed)
    imgs = [Image.fromarray(rng.integers(0, 256, (240, 240, 3), dtype=np.uint8)) for _ in range(n)]
    sizes = [(int(rng.integers(100, 900)), int(rng.integers(100, 900))) for _ in range(n)]
    return imgs, sizes


class _StandOwl:
    """ReRankerOwl's surface as the subclass uses it, over n hits with one image each."""
    images, sizes = None, None

    def __init__(self, model_name, device, image_size):
        self.model_name, self.device, self.image_size = model_name, device, image_size
        self.model = None
        self._model_map = {model_name: model_name}

    def format_results(self, results, searchable_fields=None):
        import pandas as pd
        rows = [{"_rerank_id": i, "field_content": f"img{i}.png", "original_field_name": "image"}
                for i in range(len(results["hits"]))]
        self.formatted_results = types.SimpleNamespace(
            results_df=pd.DataFrame(rows),
            format_for_model=lambda df, attrs, query: df.assign(query=query)[
                ["query", "field_content", "original_field_name", "_rerank_id"]])

    @staticmethod
    def _prepare_inputs(df):
        return df[["query", "field_content"]].values.tolist()

    def load_images(self, names, size):
        idx = [int(n[3:-4]) for n in names]
        return tuple(self.images[i] for i in idx), tuple(self.sizes[i] for i in idx)

    def get_reranked_results(self, highlight_content_column="field_content"):
        self.highlight_column = highlight_content_column


class _OracleDetector:
    """The oracle behind the B200OwlDetector.detect surface, at image size 240 (no squash)."""

    def __init__(self, sd, arch, ids):
        self.sd, self.arch, self.ids, self.calls = sd, arch, ids, 0

    def raw(self, images):
        hwc = np.stack([np.asarray(im) for im in images])
        return O.detect(self.sd, O.pixels_from_u8(hwc), self.ids, self.arch["vision"]["heads"],
                        self.arch["text"]["heads"])

    def detect(self, query, images):
        self.calls += 1
        logits, boxes = self.raw(images)
        return [O.post_process(logits[i], boxes[i], 240, 240) for i in range(len(images))]


@pytest.mark.parametrize("num_highlights", [1, 3])
def test_served_rerank_matches_reference_loop(num_highlights):
    from marqo_b200 import weights as W
    from marqo_b200.owl_reranker import make_owl_reranker_class
    arch = _arch(128, 1, 2, 16, 240, 128)
    sd = W.random_owlvit_weights(arch, 11)
    ids = np.zeros(16, np.int64)
    ids[:4] = [998, 5, 77, 999]
    det = _OracleDetector(sd, arch, ids)
    imgs, sizes = _images(5, 2)
    cx = _helpers()
    cls = make_owl_reranker_class(_StandOwl, cx, None)
    r = cls("owl/ViT-B/32", "cuda", (240, 240))
    r.model, r.images, r.sizes = det, imgs, sizes
    _StandOwl.images, _StandOwl.sizes = imgs, sizes
    r.rerank("a cat", {"hits": [{} for _ in imgs]}, ["image"], num_highlights=num_highlights)
    assert det.calls == 1
    # the reference's loop: one image per forward, then post_process, sort, top-k and rescale per image
    _b, _s, _i, _bo = [], [], [], []
    for i, im in enumerate(imgs):
        logits, boxes = det.raw([im])
        scores, corners = O.post_process(logits[0], boxes[0], 240, 240)
        b, s, ident = cx.sort_owl_boxes_scores(corners, scores, [f"img{i}.png"] * len(scores))
        b, s, ident = b[:num_highlights], s[:num_highlights], ident[:num_highlights]
        _bo += [cx.image_processor.rescale_box(x.tolist(), (240, 240), sizes[i]) for x in b]
        _b.append(b)
        _s.append(s)
        _i += ident
    torch.testing.assert_close(r.boxes, torch.cat(_b), rtol=1e-5, atol=1e-4)
    torch.testing.assert_close(r.scores, torch.cat(_s), rtol=1e-5, atol=1e-6)
    assert r.identifier == _i
    np.testing.assert_allclose(np.asarray(r.boxes_original), np.asarray(_bo), rtol=1e-5, atol=1e-3)
    assert r.inputs_df["field_content"].tolist() == _i
    assert r.highlight_column == "bbox_original"
