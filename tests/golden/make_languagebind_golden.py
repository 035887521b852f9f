"""Generate tests/golden/languagebind_golden.npz by RUNNING THE REFERENCE'S OWN CODE (the Marqo source tree that
_reference_import.REFERENCE_SRC names; the tests read only the committed fixture).

What is executed from the reference (via the import shim in _reference_import.py):
  * languagebind/video/modeling_video.py: LanguageBindVideo at a small seeded config (width 128, two heads of 64, two
    layers, 8 frames, 56 px, patch 14; a 128-wide causal text tower over 16 positions), in both embedding forms
    (clip_type "vl": CLIPVisionEmbeddings, "vl_new": CLIPVisionEmbeddings3D with tube 1) and both activations
    (quick_gelu, gelu).  Its vision_model and visual_projection encode two videos of transformed frames, its
    text_model and text_projection three token rows.  The weights are marqo_b200.weights.
    random_languagebind_video_weights at the seeds recorded in the fixture.
  The video module is imported as a package of its own directory: languagebind/__init__.py imports the audio tower,
  which needs torchaudio.  The outputs get LanguageBind.forward's rule (languagebind/__init__.py:55-64: v / |v|, times
  exp(logit_scale) for the video) without Marqo's extra normalisation.
  transformers 5.5's CLIPAttention.forward takes (hidden_states, attention_mask, **kwargs) and drops the
  causal_attention_mask the reference's CLIPEncoderLayer passes (modeling_video.py:245-250), so its text tower would
  run without the causal mask; the text layers' attention is wrapped to add that mask to the logits as the pinned
  transformers 4.41.2's CLIPAttention does.

Caveat recorded in the fixture: transformers here is 5.5.0 (the reference pins 4.41.2), torch 2.11 (pins 1.12.1).

Run:  python tests/golden/make_languagebind_golden.py
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)

import _reference_import as RI  # noqa: E402

RI.install()
import torch  # noqa: E402
import transformers  # noqa: E402

from marqo_b200 import weights as W  # noqa: E402

VIDEO_DIR = os.path.join(RI.REFERENCE_SRC, "marqo", "s2_inference", "languagebind", "video")
pkg = types.ModuleType("languagebind_video")
pkg.__path__ = [VIDEO_DIR]
sys.modules["languagebind_video"] = pkg
from languagebind_video.configuration_video import LanguageBindVideoConfig  # noqa: E402
from languagebind_video.modeling_video import LanguageBindVideo  # noqa: E402

ARCH = {"embed_dim": 64, "video_frames": 8,
        "vision": {"width": 128, "layers": 2, "heads": 2, "mlp": 512, "patch": 14, "image_size": 56},
        "text": {"width": 128, "layers": 2, "heads": 2, "mlp": 512, "ctx": 16, "vocab": 1000}}
CASES = [("vl", "quick_gelu", 11), ("vl_new", "quick_gelu", 12), ("vl", "gelu", 13), ("vl_new", "gelu", 14)]


def config(form, act):
    v, t = ARCH["vision"], ARCH["text"]
    return LanguageBindVideoConfig(
        projection_dim=ARCH["embed_dim"],
        text_config=dict(hidden_size=t["width"], intermediate_size=t["mlp"], num_hidden_layers=t["layers"],
                         num_attention_heads=t["heads"], max_position_embeddings=t["ctx"], vocab_size=t["vocab"],
                         hidden_act=act),
        vision_config=dict(hidden_size=v["width"], intermediate_size=v["mlp"], num_hidden_layers=v["layers"],
                           num_attention_heads=v["heads"], image_size=v["image_size"], patch_size=v["patch"],
                           hidden_act=act, add_time_attn=True, num_frames=ARCH["video_frames"], clip_type=form,
                           tube_size=1, force_patch_dropout=0.0, video_decode_backend="opencv"))


T, S = ARCH["video_frames"], ARCH["vision"]["image_size"]
PIXEL_SEED = 2025   # the test regenerates the pixels: default_rng(PIXEL_SEED).standard_normal((2, T, 3, S, S))
pixels = np.random.default_rng(PIXEL_SEED).standard_normal((2, T, 3, S, S)).astype(np.float32)
rng = np.random.default_rng(7)
ids = np.zeros((3, ARCH["text"]["ctx"]), np.int64)
for r, n in enumerate((5, 16, 9)):
    ids[r, :n] = rng.integers(1, 998, n)
    ids[r, n - 1] = 999            # EOT: the largest id
ids[2, 9:] = 999                   # padded with EOT, as LanguageBindVideoTokenizer pads: the first arg-max is pooled
out = {"pixel_seed": np.int64(PIXEL_SEED), "ids": ids.astype(np.int32), "forms": np.array([c[0] for c in CASES]),
       "acts": np.array([c[1] for c in CASES]), "seeds": np.array([c[2] for c in CASES], np.int64),
       "versions": np.array([transformers.__version__, torch.__version__])}
for j, (form, act, seed) in enumerate(CASES):
    model = LanguageBindVideo(config(form, act)).eval()
    sd = W.random_languagebind_video_weights(ARCH, seed, form=form)
    missing, unexpected = model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()},
                                                strict=False)
    assert not unexpected and all(k.endswith("position_ids") for k in missing), (missing, unexpected)
    for layer in model.text_model.encoder.layers:
        attn_forward = layer.self_attn.forward

        def causal_forward(hidden_states, attention_mask=None, causal_attention_mask=None, _f=attn_forward, **kw):
            if causal_attention_mask is not None:
                attention_mask = causal_attention_mask if attention_mask is None else attention_mask + causal_attention_mask
            return _f(hidden_states, attention_mask=attention_mask, **kw)

        layer.self_attn.forward = causal_forward
    with torch.no_grad():
        pv = torch.from_numpy(pixels).permute(0, 2, 1, 3, 4)   # [B, C, T, H, W], as the processor returns it
        v = model.visual_projection(model.vision_model(pv)[1])
        v = v / v.norm(p=2, dim=-1, keepdim=True) * model.logit_scale.exp()
        t = model.text_projection(model.text_model(torch.from_numpy(ids))[1])
        t = t / t.norm(p=2, dim=-1, keepdim=True)
    out[f"video_{j}"] = v.numpy()
    out[f"text_{j}"] = t.numpy()
np.savez_compressed(os.path.join(HERE, "languagebind_golden.npz"), **out)
print("wrote languagebind_golden.npz", {k: v.shape for k, v in out.items()})
