"""Model name -> properties + architecture for the models the engine serves.

Property dicts (`name`, `dimensions`, `type`, `tokens`, `model_size`, prefixes, `poolingMethod`, `notes`) are the
reference's registry entries (src/marqo/s2_inference/model_registry.py:142-231 for open_clip/*, :616-851 for hf/*);
`type` is rewritten to the engine's loader types ("b200_open_clip" / "b200_hf" / "b200_hf_stella") so that both
engines can be registered side by side in MODEL_PROPERTIES['loaders'] (model_registry.py:2133-2145).  The `arch` blocks are the shapes that live
in open_clip 2.24.0 `model_configs/*.json` and the HF `config.json` files (SURVEY.md §8).

The hf/* shapes come from the upstream HF `config.json` files, which cannot be re-read offline (like the ViT shapes of
SURVEY.md §8).  All are uncased-WordPiece BERTs (vocabulary 30522, 512 positions, 2 token types, erf-GELU, mlp = 4 x
width), mean-pooled:
    MiniLM-L6  (all-MiniLM-L6-v1/v2, all_datasets_v3/v4_MiniLM-L6)                 width  384, 6 layers, 12 heads
    MiniLM-L12 (all_datasets_v3/v4_MiniLM-L12)                                      width  384, 12 layers, 12 heads
    e5-small, e5-small-v2, e5-small-unsupervised, bge-small-en-v1.5                width  384, 12 layers, 12 heads
    e5-base, e5-base-v2, e5-base-unsupervised, bge-base-en-v1.5                    width  768, 12 layers, 12 heads
    e5-large, e5-large-v2, e5-large-unsupervised, bge-large-en-v1.5                width 1024, 24 layers, 16 heads
The 384-wide models have head_dim 32, the others head_dim 64.

The MPNet entries (all-mpnet-base-v1/v2, all_datasets_v3/v4_mpnet-base; model_registry.py:630-641,668-679) live in a
table of their own, MPNET_MODELS, behind `find_model` / `all_models`: they are MPNet-base checkpoints (`arch["kind"] ==
"mpnet"`), which the same `b200_hf` loader serves with the MPNet runtime and tokenizer.  Their shapes come from the
upstream config.json files and cannot be re-read offline (verify): width 768, 12 layers, 12 heads, mlp 3072, vocabulary
30527, max_position_embeddings 514 (positions start after pad_token_id 1, so at most 512 tokens), layer_norm_eps 1e-5
(MPNetConfig's default is 1e-12), 32 relative-attention buckets with max distance 128, mean pooling.

The SigLIP entries (model_registry.py:385-433,489-494) live in SIGLIP_MODELS (`arch["kind"] == "siglip"`), served by
the same `b200_open_clip` loader.  Their shapes come from open_clip 2.24.0's model_configs/ViT-{B,L}-16-SigLIP*.json,
`pretrained._slpcfg` and timm's `AttentionPoolLatent`, none of which can be re-read offline (verify):
    ViT-B-16-SigLIP{,-256,-384,-512}/webli, Marqo/marqo-fashionSigLIP
        vision: timm vit_base_patch16_siglip_*: width 768, 12 layers, 12 heads, mlp 3072, patch 16, image 224 / 256 /
        384 / 512 (fashionSigLIP: 224); text: width 768, 12 layers, 12 heads, mlp 3072, ctx 64, vocab 32000; embed 768
    ViT-L-16-SigLIP-256/webli, ViT-L-16-SigLIP-384/webli
        vision: width 1024, 24 layers, 16 heads, mlp 4096, patch 16, image 256 / 384; text: width 1024, 24 layers,
        16 heads, mlp 4096, ctx 64, vocab 32000; embed 1024
    Both towers: pre-LN blocks, LayerNorm eps 1e-6, erf-GELU.  Vision: no class token, patch conv with bias, no ln_pre,
    final LN over all tokens, then the MAP head (a learned latent query attends over the tokens, proj, x + MLP(LN(x)),
    MLP 4 x width); no projection (timm_proj "none").  Text: no causal mask, ln_final, last position pooled, Linear with
    bias (proj_bias).  Preprocessing (_slpcfg): mean = std = 0.5, bicubic squash resize to S x S without a crop.
ViT-SO400M-14-SigLIP-384 (width 1152, 16 heads: head_dim 72) is not served.

The multilingual-e5 entries (model_registry.py:735-760,788-794) live in XLMR_MODELS, served by the `b200_hf` loader
with the SentencePiece Unigram tokenizer of XLM-RoBERTa (fairseq id offset: <s> 0, <pad> 1, </s> 2, <unk> 3, every
other piece at its SentencePiece id + 1).  Their shapes come from the upstream config.json files and cannot be re-read
offline (verify):
    multilingual-e5-base              XLMRobertaModel (`arch["kind"] == "xlmr"`): width 768, 12 layers, 12 heads,
                                      mlp 3072, vocabulary 250002, max_position_embeddings 514 (positions start after
                                      pad_token_id 1, so at most 512 tokens), one token type, layer_norm_eps 1e-5
    multilingual-e5-large{,-instruct} the same at width 1024, 24 layers, 16 heads, mlp 4096
    multilingual-e5-small             a BertModel (Multilingual-MiniLM-L12-H384, `arch["kind"]` absent): width 384,
                                      12 layers, 12 heads, mlp 1536, vocabulary 250037, 512 positions, 2 token types,
                                      layer_norm_eps 1e-12; it runs the BERT runtime unchanged
All four mean-pool the last hidden state and erf-GELU their MLPs.

The OpenAI ResNet CLIP entries (model_registry.py:80-126) live in RESNET_MODELS (`arch["kind"] == "clip_resnet"`),
served by the `b200_open_clip` loader.  Their shapes come from open_clip 2.24.0's model_configs/RN50.json, RN101.json
and `ModifiedResNet`, which cannot be re-read offline (verify): image 224, width 64, stages of [3, 4, 6, 3] (RN50) or
[3, 4, 23, 3] (RN101) Bottlenecks, a 7 x 7 x 2048 trunk output and an attention pool of 32 heads (head_dim 64) whose
output is embed_dim wide (1024 / 512); the CLIP text tower (width 512, 12 layers, 8 heads, mlp 2048, ctx 77, vocab
49408).  Every `openai` tag loads as QuickGELU (as ViT-B-32/openai does here), the `-quickgelu` names too; the
yfcc15m / cc12m tags of the plain names run erf-GELU.  OpenAI mean and std, shortest side -> 224 + centre crop.  The
arch block has no "vision" key: the text tower's fields sit at the top level, as in the BERT archs, and the CNN in its
own "resnet" block.

The ConvNeXt CLIP entries (model_registry.py:274-343) live in CONVNEXT_MODELS (`arch["kind"] == "clip_convnext"`),
served by the `b200_open_clip` loader, in the clip_resnet layout with the trunk in a "convnext" block.  find_model
finds them; all_models() leaves them out (see there).  Their shapes
come from open_clip 2.24.0's model_configs/convnext_*.json, its `TimmModel` and timm's convnext.py, none of which can
be re-read offline (verify):
    convnext_base        timm convnext_base: dims 128, 256, 512, 1024, depths 3, 3, 27, 3; image 224; linear head;
                         text width 512, 8 heads, 12 layers
    convnext_base_w      the same trunk at image 256; text width 640, 10 heads, 12 layers
    convnext_base_w_320  convnext_base_w at image 320
    convnext_large_d     timm convnext_large: dims 192, 384, 768, 1536, depths 3, 3, 27, 3; image 256; MLP head
                         (fc1 with bias to 2 embed, GELU, fc2 without bias); text width 768, 12 heads, 16 layers
    convnext_large_d_320 convnext_large_d at image 320
    convnext_xxlarge     timm convnext_xxlarge: dims 384, 768, 1536, 3072, depths 3, 4, 30, 3; image 256; linear
                         head; trunk LayerNorm eps 1e-5 (timm's norm_eps for this model; 1e-6 for the others); text
                         width 1024, 16 heads, 24 layers
The heads pool with timm's own head (global average pool, then its LayerNorm), and the Linear head has no bias.  Every
text tower has mlp 4 width, ctx 77, vocabulary 49408 and erf-GELU, as do the trunk's MLPs.  OpenAI mean and std,
shortest side -> S + centre crop, as for CLIP (not SigLIP's squash).

The big open_clip ViTs (model_registry.py:237-256,378-384,392-398) live in BIG_VIT_MODELS, in the CLIP layout of
MODELS, served by the `b200_open_clip` loader.  find_model finds them; all_models() leaves them out (see there).
Their shapes come from open_clip 2.24.0's model_configs/ViT-{H,g,bigG}-14*.json (head_width, mlp_ratio 4.3637 for g
and 4.9231 for bigG) and their DFN5B preprocessing from its pretrained.py, none of which can be re-read offline
(verify):
    ViT-H-14/laion2b_s32b_b79k          vision width 1280, 32 layers, 16 heads (head_dim 80), mlp 5120, image 224;
                                        text width 1024, 24 layers, 16 heads, mlp 4096; embed 1024; erf-GELU
    ViT-H-14-quickgelu/dfn5b            the same with QuickGELU and the bicubic squash resize (resize_mode "squash")
    ViT-H-14-378-quickgelu/dfn5b        ViT-H-14-quickgelu/dfn5b at image 378 (27 x 27 + 1 = 730 tokens)
    ViT-g-14/laion2b_s{12b_b42k,34b_b88k} vision width 1408, 40 layers, 16 heads (head_dim 88), mlp 6144, image 224;
                                        text as ViT-H-14; embed 1024; erf-GELU
    ViT-bigG-14/laion2b_s39b_b160k      vision width 1664, 48 layers, 16 heads (head_dim 104), mlp 8192, image 224;
                                        text width 1280, 32 layers, 20 heads, mlp 5120; embed 1280; erf-GELU
All use patch 14, the class token, ln_pre / ln_post, LayerNorm eps 1e-5, OpenAI mean and std, ctx 77, vocabulary
49408 and the causal CLIP text tower.  The vision heads of 80, 88 and 104 run zero-padded to the attention kernel's
96, 96 and 128.  The entries carry no model_size: Marqo derives 5, 5 and 6 GB from the names.  ViT-SO400M-14-SigLIP-384
(head_dim 72) and xlm-roberta-large-ViT-H-14 are not served.

The EVA02 CLIP entries (model_registry.py:441-461) live in EVA02_MODELS (`arch["kind"] == "clip_eva"`), served by the
`b200_open_clip` loader, in the clip_resnet layout: the text tower's fields at the top level and the trunk in an "eva"
block.  Their shapes come from open_clip 2.24.0's model_configs/EVA02-*.json, its `TimmModel` / `CustomTextCLIP` and
timm's eva.py (`Eva`, `EvaAttention`, `SwiGLU`, `RotaryEmbeddingCat`), none of which can be re-read offline (verify):
    EVA02-B-16/merged2b_s8b_b131k      trunk width 768, 12 layers, 12 heads, SwiGLU hidden 2048, patch 16, image 224
                                       (197 tokens); text width 512, 12 layers, 8 heads; embed 512
    EVA02-L-14/merged2b_s4b_b131k      trunk width 1024, 24 layers, 16 heads, SwiGLU hidden 2730, patch 14, image 224
                                       (257 tokens); text width 768, 12 layers, 12 heads; embed 768
    EVA02-L-14-336/merged2b_s6b_b61k   EVA02-L-14 at image 336 (577 tokens)
The hidden size is int(width * 4 * 2 / 3).  Every head is 64 wide; every trunk LayerNorm has eps 1e-6.  The trunk:
    x = [cls_token ; patch_embed(img) + its bias] + pos_embed            (no ln_pre, no layer scale)
    per block:  h = norm1(x);  q = h Wq^T + bq,  k = h Wk^T (no bias),  v = h Wv^T + bv
                q and k of tokens 1..N-1 rotated (RoPE below), token 0 not;  o = softmax(q k^T / 8) v per head
                x += attn.proj(attn.norm(o))                            (LayerNorm over the full width of o)
                h = norm2(x);  u = SiLU(h Wg^T + bg) * (h Wx^T + bx)
                x += mlp.fc2(mlp.norm(u))                               (LayerNorm over the hidden row)
    out = head(norm(x)[token 0]), head a Linear [E, W] with bias, then the CLIP L2 rule (no epsilon).
RoPE (timm build_fourier_pos_embed with the "ij" grid, repeat_interleave(2), apply_rot_embed_cat; in_pixels False,
ref_feat_shape (16, 16)): the patch at grid row r and column c is token 1 + r G + c, s = 16 / G.  Pair i = 0..31 of
a head (columns 2i, 2i + 1) turns by theta = p 10000^(-j/16), j = i mod 16, p = r s for i < 16 and c s for i >= 16:
(a, b) -> (a cos - b sin, b cos + a sin).  The table is a non-persistent buffer, so the engine builds it.  The text
tower is the causal CLIP tower (erf-GELU, LayerNorm eps 1e-5, ctx 77, vocabulary 49408, EOT pooling, ln_final, a
[W, E] projection without bias) under the "text." prefix.  OpenAI mean and std, shortest side -> S + centre crop.  The
entries carry no model_size: Marqo derives 1 GB from the open_clip type.

The Stella embedder Marqo/dunzhang-stella_en_400M_v5 (model_registry.py:898-904) lives in GTE_MODELS (`arch["kind"] ==
"gte"`), served by its own loader type "b200_hf_stella" (the reference's "hf_stella": HuggingFaceStellaModel, a
HuggingFaceModel that requires trustRemoteCode and loads with use_memory_efficient_attention False and unpad_inputs
False).  The checkpoint is Alibaba's NewModel (the gte-v1.5 architecture, trust_remote_code).  Its shapes come from
its config.json and modeling.py, which cannot be re-read offline (verify): width 1024, 24 layers, 16 heads (head_dim
64), GeGLU hidden 4096, vocabulary 30528, 2 token types, erf-GELU, LayerNorm eps 1e-12, position_embedding_type "rope"
with rope_theta 160000 and rope_scaling {type "ntk", factor 2.0}, max_position_embeddings 8192, no logn attention
scale; mean pooling of the last hidden state (no 2_Dense projection), then F.normalize.  Over right-padded ids:
    x = LN_emb(word[ids] + token_type[0])                               (no position table)
    per layer (post-LN):  q | k | v = x Wqkv^T + bqkv;  q, k rotated by position s (RoPE below)
                          x = attn_ln(x + attention(q, k, v) Wo^T + bo)  (padded keys masked, scale 1/8)
                          up | gate = x Wug^T (no bias);  x = mlp_ln(x + (GELU(gate) * up) Wd^T + bd)
RoPE (NTKScalingRotaryEmbedding, rotate_half): the cache is built at 8192 * 2 positions, beyond
max_position_embeddings, so the NTK branch applies: pair j = 0..31 of a head (columns j and j + 32) turns by s f_j,
f_j = (160000 * 2)^(-2j/64) / 2^(2/64): (a, b) -> (a cos - b sin, b cos + a sin).  The uncased BERT WordPiece
tokenizer ([CLS] 101, [SEP] 102, pad 0) is the engine's WordPieceTokenizer.  The entry carries no model_size: Marqo
has no size for the hf_stella type and takes its default, 0.66 GB."""
from __future__ import annotations

import copy
from typing import Dict, Optional

OPENAI_MEAN = (0.48145466, 0.4578275, 0.40821073)   # src/marqo/s2_inference/clip_utils.py:32-33
OPENAI_STD = (0.26862954, 0.26130258, 0.27577711)

TYPE_OPEN_CLIP = "b200_open_clip"
TYPE_HF = "b200_hf"
TYPE_HF_STELLA = "b200_hf_stella"


def _clip_arch(embed, vw, vl, vh, patch, tw, tl, th, act="gelu"):
    return {
        "embed_dim": embed, "act": act, "mean": OPENAI_MEAN, "std": OPENAI_STD,
        "vision": {"width": vw, "layers": vl, "heads": vh, "mlp": 4 * vw, "patch": patch, "image_size": 224},
        "text": {"width": tw, "layers": tl, "heads": th, "mlp": 4 * tw, "ctx": 77, "vocab": 49408},
    }


def _bert_arch(w, layers, heads, pool="mean"):
    return {"width": w, "layers": layers, "heads": heads, "mlp": 4 * w, "vocab": 30522, "max_pos": 512,
            "type_vocab": 2, "pool": pool}


_VIT_B_32 = dict(embed=512, vw=768, vl=12, vh=12, patch=32, tw=512, tl=12, th=8)
_VIT_B_16 = dict(embed=512, vw=768, vl=12, vh=12, patch=16, tw=512, tl=12, th=8)
_VIT_L_14 = dict(embed=768, vw=1024, vl=24, vh=16, patch=14, tw=768, tl=12, th=12)


# (width, layers, heads) of the hf/* BERTs (module docstring)
_MINILM_L6 = (384, 6, 12)
_MINILM_L12 = (384, 12, 12)
_BERT_SMALL = (384, 12, 12)
_BERT_BASE = (768, 12, 12)
_BERT_LARGE = (1024, 24, 16)
_BGE_QUERY_PREFIX = "Represent this sentence for searching relevant passages: "


def _hf(name: str, tokens: int, shape: tuple, **props) -> dict:
    """A reference hf/* entry (`dimensions` = width: every one of them mean-pools the last hidden state) + its arch."""
    return {"name": name, "dimensions": shape[0], "tokens": tokens, "type": TYPE_HF, **props, "notes": "",
            "arch": _bert_arch(*shape)}


def _open_clip(name: str, dims: int, pretrained: str, shape: dict, act: str) -> dict:
    return {"name": name, "dimensions": dims, "note": "open_clip models", "type": TYPE_OPEN_CLIP,
            "pretrained": pretrained, "arch": _clip_arch(**shape, act=act)}


def _models() -> Dict[str, dict]:
    m: Dict[str, dict] = {}
    for tag in ("laion400m_e31", "laion400m_e32", "laion2b_e16", "laion2b_s34b_b79k"):
        m[f"open_clip/ViT-B-32/{tag}"] = _open_clip(f"open_clip/ViT-B-32/{tag}", 512, tag, _VIT_B_32, "gelu")
    m["open_clip/ViT-B-32/openai"] = _open_clip("open_clip/ViT-B-32/openai", 512, "openai", _VIT_B_32, "quickgelu")
    m["open_clip/ViT-B-32-quickgelu/openai"] = _open_clip("open_clip/ViT-B-32-quickgelu/openai", 512, "openai",
                                                          _VIT_B_32, "quickgelu")
    m["open_clip/ViT-B-16/openai"] = _open_clip("open_clip/ViT-B-16/openai", 512, "openai", _VIT_B_16, "quickgelu")
    m["open_clip/ViT-B-16/laion2b_s34b_b88k"] = _open_clip("open_clip/ViT-B-16/laion2b_s34b_b88k", 512,
                                                           "laion2b_s34b_b88k", _VIT_B_16, "gelu")
    for tag in ("laion400m_e31", "laion400m_e32", "laion2b_s32b_b82k"):
        m[f"open_clip/ViT-L-14/{tag}"] = _open_clip(f"open_clip/ViT-L-14/{tag}", 768, tag, _VIT_L_14, "gelu")
    m["open_clip/ViT-L-14/openai"] = _open_clip("open_clip/ViT-L-14/openai", 768, "openai", _VIT_L_14, "quickgelu")
    # (verify) upstream uses 0.5/0.5 image statistics for this tag (SURVEY.md Appendix B)
    m["open_clip/ViT-L-14/laion2b_s32b_b82k"]["arch"]["mean"] = (0.5, 0.5, 0.5)
    m["open_clip/ViT-L-14/laion2b_s32b_b82k"]["arch"]["std"] = (0.5, 0.5, 0.5)
    for short, repo, tokens, shape in (("all-MiniLM-L6-v1", "sentence-transformers/all-MiniLM-L6-v1", 128, _MINILM_L6),
                                       ("all-MiniLM-L6-v2", "sentence-transformers/all-MiniLM-L6-v2", 256, _MINILM_L6),
                                       ("all_datasets_v3_MiniLM-L12", "flax-sentence-embeddings/all_datasets_v3_MiniLM-L12",
                                        128, _MINILM_L12),
                                       ("all_datasets_v3_MiniLM-L6", "flax-sentence-embeddings/all_datasets_v3_MiniLM-L6",
                                        128, _MINILM_L6),
                                       ("all_datasets_v4_MiniLM-L12", "flax-sentence-embeddings/all_datasets_v4_MiniLM-L12",
                                        128, _MINILM_L12),
                                       ("all_datasets_v4_MiniLM-L6", "flax-sentence-embeddings/all_datasets_v4_MiniLM-L6",
                                        128, _MINILM_L6)):
        m[f"hf/{short}"] = _hf(repo, tokens, shape)
    for short, tokens, size, shape in (("e5-small", 192, 0.1342, _BERT_SMALL),
                                       ("e5-base", 192, 0.438, _BERT_BASE),
                                       ("e5-large", 192, 1.3, _BERT_LARGE),
                                       ("e5-large-unsupervised", 128, 1.3, _BERT_LARGE),
                                       ("e5-base-unsupervised", 128, 0.438, _BERT_BASE),
                                       ("e5-small-unsupervised", 128, 0.134, _BERT_SMALL),
                                       ("e5-small-v2", 512, 0.134, _BERT_SMALL),
                                       ("e5-base-v2", 512, 0.438, _BERT_BASE),
                                       ("e5-large-v2", 512, 1.34, _BERT_LARGE)):
        m[f"hf/{short}"] = _hf(f"intfloat/{short}", tokens, shape, model_size=size, text_query_prefix="query: ",
                               text_chunk_prefix="passage: ")
    for size, shape in (("small", _BERT_SMALL), ("base", _BERT_BASE), ("large", _BERT_LARGE)):
        m[f"hf/bge-{size}-en-v1.5"] = _hf(f"BAAI/bge-{size}-en-v1.5", 512, shape, text_query_prefix=_BGE_QUERY_PREFIX,
                                          poolingMethod="mean")
    return m


MODELS: Dict[str, dict] = _models()


def _mpnet_arch() -> dict:
    """MPNet-base (module docstring, verify)."""
    return {"kind": "mpnet", "width": 768, "layers": 12, "heads": 12, "mlp": 3072, "vocab": 30527, "max_pos": 514,
            "pad_id": 1, "ln_eps": 1e-5, "rel_buckets": 32, "rel_max_distance": 128, "pool": "mean"}


def _mpnet_models() -> Dict[str, dict]:
    m: Dict[str, dict] = {}
    for short, repo in (("all-mpnet-base-v1", "sentence-transformers/all-mpnet-base-v1"),
                        ("all-mpnet-base-v2", "sentence-transformers/all-mpnet-base-v2"),
                        ("all_datasets_v3_mpnet-base", "flax-sentence-embeddings/all_datasets_v3_mpnet-base"),
                        ("all_datasets_v4_mpnet-base", "flax-sentence-embeddings/all_datasets_v4_mpnet-base")):
        m[f"hf/{short}"] = {"name": repo, "dimensions": 768, "tokens": 128, "type": TYPE_HF, "notes": "",
                            "arch": _mpnet_arch()}
    return m


MPNET_MODELS: Dict[str, dict] = _mpnet_models()

SIGLIP_MEAN = (0.5, 0.5, 0.5)   # open_clip pretrained._slpcfg (verify)
SIGLIP_STD = (0.5, 0.5, 0.5)


def _siglip_arch(w: int, layers: int, heads: int, image_size: int) -> dict:
    """SigLIP ViT-{B,L}-16 (module docstring, verify): both towers share width, depth and heads."""
    return {
        "kind": "siglip", "embed_dim": w, "act": "gelu", "mean": SIGLIP_MEAN, "std": SIGLIP_STD,
        "resize_mode": "squash", "ln_eps": 1e-6,
        "vision": {"width": w, "layers": layers, "heads": heads, "mlp": 4 * w, "patch": 16, "image_size": image_size,
                   "map_mlp": 4 * w},
        "text": {"width": w, "layers": layers, "heads": heads, "mlp": 4 * w, "ctx": 64, "vocab": 32000},
    }


def _siglip_models() -> Dict[str, dict]:
    m: Dict[str, dict] = {}
    shapes = [(f"ViT-B-16-SigLIP{suffix}", 768, 12, 12, size)
              for suffix, size in (("", 224), ("-256", 256), ("-384", 384), ("-512", 512))]
    shapes += [(f"ViT-L-16-SigLIP-{size}", 1024, 24, 16, size) for size in (256, 384)]
    for model, w, layers, heads, size in shapes:
        name = f"open_clip/{model}/webli"
        m[name] = {"name": name, "dimensions": w, "note": f"open_clip model: {model}/webli", "type": TYPE_OPEN_CLIP,
                   "pretrained": "webli", "arch": _siglip_arch(w, layers, heads, size)}
    # model_registry.py:489-494: an hf-hub open_clip model, no `pretrained` tag
    m["Marqo/marqo-fashionSigLIP"] = {"name": "hf-hub:Marqo/marqo-fashionSigLIP", "dimensions": 768,
                                      "note": "Marqo's fashionSigLIP model", "type": TYPE_OPEN_CLIP,
                                      "arch": _siglip_arch(768, 12, 12, 224)}
    return m


SIGLIP_MODELS: Dict[str, dict] = _siglip_models()


_E5_INSTRUCT_QUERY_PREFIX = "Instruct: Given a web search query, retrieve relevant passages that answer the query\nQuery: "


def _xlmr_arch(w: int, layers: int, heads: int) -> dict:
    """XLMRobertaModel (module docstring, verify)."""
    return {"kind": "xlmr", "width": w, "layers": layers, "heads": heads, "mlp": 4 * w, "vocab": 250002, "max_pos": 514,
            "pad_id": 1, "type_vocab": 1, "ln_eps": 1e-5, "pool": "mean"}


def _xlmr_models() -> Dict[str, dict]:
    m: Dict[str, dict] = {}
    # Multilingual-MiniLM-L12-H384: a BertModel over the XLM-R SentencePiece vocabulary (module docstring, verify)
    small = {**_bert_arch(*_BERT_SMALL), "vocab": 250037, "tokenizer": "xlmr"}
    e5 = {"text_query_prefix": "query: ", "text_chunk_prefix": "passage: "}
    for short, arch, props in (
            ("multilingual-e5-small", small, {"model_size": 0.471, **e5}),
            ("multilingual-e5-base", _xlmr_arch(768, 12, 12), {"model_size": 1.11, **e5}),
            ("multilingual-e5-large", _xlmr_arch(1024, 24, 16), {"model_size": 2.24, **e5}),
            ("multilingual-e5-large-instruct", _xlmr_arch(1024, 24, 16),
             {"text_query_prefix": _E5_INSTRUCT_QUERY_PREFIX})):
        m[f"hf/{short}"] = {"name": f"intfloat/{short}", "dimensions": arch["width"], "tokens": 512, "type": TYPE_HF,
                            **props, "notes": "", "arch": arch}
    return m


XLMR_MODELS: Dict[str, dict] = _xlmr_models()


def _resnet_arch(layers: list, embed: int, act: str) -> dict:
    """OpenAI ResNet CLIP (module docstring, verify)."""
    return {"kind": "clip_resnet", "embed_dim": embed, "act": act, "mean": OPENAI_MEAN, "std": OPENAI_STD,
            "width": 512, "layers": 12, "heads": 8, "mlp": 2048, "ctx": 77, "vocab": 49408,
            "resnet": {"layers": list(layers), "width": 64, "heads": 32, "image_size": 224}}


def _resnet_models() -> Dict[str, dict]:
    m: Dict[str, dict] = {}
    for model, layers, embed, tags in (("RN50", [3, 4, 6, 3], 1024, ("openai", "yfcc15m", "cc12m")),
                                       ("RN101", [3, 4, 23, 3], 512, ("openai", "yfcc15m"))):
        for variant in (model, f"{model}-quickgelu"):
            for tag in tags:
                act = "quickgelu" if tag == "openai" or variant.endswith("-quickgelu") else "gelu"
                name = f"open_clip/{variant}/{tag}"
                m[name] = {"name": name, "dimensions": embed, "note": "open_clip models", "type": TYPE_OPEN_CLIP,
                           "pretrained": tag, "arch": _resnet_arch(layers, embed, act)}
    return m


RESNET_MODELS: Dict[str, dict] = _resnet_models()


def _convnext_arch(trunk: str, image: int, head: str, embed: int, tw: int, tl: int, th: int) -> dict:
    """ConvNeXt CLIP (module docstring, verify)."""
    dims, depths, eps = {"base": ([128, 256, 512, 1024], [3, 3, 27, 3], 1e-6),
                         "large": ([192, 384, 768, 1536], [3, 3, 27, 3], 1e-6),
                         "xxlarge": ([384, 768, 1536, 3072], [3, 4, 30, 3], 1e-5)}[trunk]
    return {"kind": "clip_convnext", "embed_dim": embed, "act": "gelu", "mean": OPENAI_MEAN, "std": OPENAI_STD,
            "width": tw, "layers": tl, "heads": th, "mlp": 4 * tw, "ctx": 77, "vocab": 49408,
            "convnext": {"dims": dims, "depths": depths, "image_size": image, "ln_eps": eps, "head": head}}


def _convnext_models() -> Dict[str, dict]:
    m: Dict[str, dict] = {}
    base_w = ("laion2b_s13b_b82k", "laion2b_s13b_b82k_augreg", "laion_aesthetic_s13b_b82k")
    for model, shape, tags in (
            ("convnext_base", ("base", 224, "linear", 512, 512, 12, 8), ("laion400m_s13b_b51k",)),
            ("convnext_base_w", ("base", 256, "linear", 640, 640, 12, 10), base_w),
            ("convnext_base_w_320", ("base", 320, "linear", 640, 640, 12, 10),
             ("laion_aesthetic_s13b_b82k", "laion_aesthetic_s13b_b82k_augreg")),
            ("convnext_large_d", ("large", 256, "mlp", 768, 768, 16, 12), ("laion2b_s26b_b102k_augreg",)),
            ("convnext_large_d_320", ("large", 320, "mlp", 768, 768, 16, 12),
             ("laion2b_s29b_b131k_ft", "laion2b_s29b_b131k_ft_soup")),
            ("convnext_xxlarge", ("xxlarge", 256, "linear", 1024, 1024, 24, 16),
             ("laion2b_s34b_b82k_augreg", "laion2b_s34b_b82k_augreg_rewind", "laion2b_s34b_b82k_augreg_soup"))):
        for tag in tags:
            name = f"open_clip/{model}/{tag}"
            m[name] = {"name": name, "dimensions": shape[3], "note": "open_clip models", "type": TYPE_OPEN_CLIP,
                       "pretrained": tag, "arch": _convnext_arch(*shape)}
    return m


CONVNEXT_MODELS: Dict[str, dict] = _convnext_models()


def _big_vit_arch(vw: int, vl: int, mlp: int, image: int, act: str, text: tuple, embed: int) -> dict:
    """ViT-H / g / bigG-14 CLIP (module docstring, verify): 16 vision heads, patch 14."""
    tw, tl, th = text
    arch = _clip_arch(embed, vw, vl, 16, 14, tw, tl, th, act=act)
    arch["vision"].update(mlp=mlp, image_size=image)
    return arch


def _big_vit_models() -> Dict[str, dict]:
    m: Dict[str, dict] = {}
    h_text, big_g_text = (1024, 24, 16), (1280, 32, 20)
    for model, tag, shape in (
            ("ViT-H-14", "laion2b_s32b_b79k", (1280, 32, 5120, 224, "gelu", h_text, 1024)),
            ("ViT-H-14-quickgelu", "dfn5b", (1280, 32, 5120, 224, "quickgelu", h_text, 1024)),
            ("ViT-H-14-378-quickgelu", "dfn5b", (1280, 32, 5120, 378, "quickgelu", h_text, 1024)),
            ("ViT-g-14", "laion2b_s12b_b42k", (1408, 40, 6144, 224, "gelu", h_text, 1024)),
            ("ViT-g-14", "laion2b_s34b_b88k", (1408, 40, 6144, 224, "gelu", h_text, 1024)),
            ("ViT-bigG-14", "laion2b_s39b_b160k", (1664, 48, 8192, 224, "gelu", big_g_text, 1280))):
        name = f"open_clip/{model}/{tag}"
        arch = _big_vit_arch(*shape)
        dfn = tag == "dfn5b"
        if dfn:
            arch["resize_mode"] = "squash"
        # the DFN5B entries have the note style of the reference's newer entries (model_registry.py:378-398)
        m[name] = {"name": name, "dimensions": shape[-1],
                   "note": f"open_clip model: {model}/{tag}" if dfn else "open_clip models", "type": TYPE_OPEN_CLIP,
                   "pretrained": tag, "arch": arch}
    return m


BIG_VIT_MODELS: Dict[str, dict] = _big_vit_models()


def _eva02_arch(embed: int, width: int, layers: int, heads: int, patch: int, image: int, text: tuple) -> dict:
    """EVA02 CLIP (module docstring, verify): the CLIP text tower at the top level, the timm Eva trunk in "eva"."""
    tw, tl, th = text
    return {"kind": "clip_eva", "embed_dim": embed, "act": "gelu", "mean": OPENAI_MEAN, "std": OPENAI_STD,
            "width": tw, "layers": tl, "heads": th, "mlp": 4 * tw, "ctx": 77, "vocab": 49408,
            "eva": {"width": width, "layers": layers, "heads": heads, "mlp": int(width * 4 * 2 / 3), "patch": patch,
                    "image_size": image, "ln_eps": 1e-6, "rope_ref_grid": 16}}


def _eva02_models() -> Dict[str, dict]:
    m: Dict[str, dict] = {}
    for model, tag, shape in (
            ("EVA02-B-16", "merged2b_s8b_b131k", (512, 768, 12, 12, 16, 224, (512, 12, 8))),
            ("EVA02-L-14", "merged2b_s4b_b131k", (768, 1024, 24, 16, 14, 224, (768, 12, 12))),
            ("EVA02-L-14-336", "merged2b_s6b_b61k", (768, 1024, 24, 16, 14, 336, (768, 12, 12)))):
        name = f"open_clip/{model}/{tag}"
        m[name] = {"name": name, "dimensions": shape[0], "note": f"open_clip model: {model}/{tag}",
                   "type": TYPE_OPEN_CLIP, "pretrained": tag, "arch": _eva02_arch(*shape)}
    return m


EVA02_MODELS: Dict[str, dict] = _eva02_models()


def _gte_arch() -> dict:
    """NewModel as the Stella embedder configures it (module docstring, verify)."""
    return {"kind": "gte", "width": 1024, "layers": 24, "heads": 16, "mlp": 4096, "vocab": 30528, "type_vocab": 2,
            "ctx": 512, "ln_eps": 1e-12, "rope_theta": 160000.0, "rope_ntk_factor": 2.0, "pool": "mean"}


GTE_MODELS: Dict[str, dict] = {
    "Marqo/dunzhang-stella_en_400M_v5": {"name": "Marqo/dunzhang-stella_en_400M_v5", "dimensions": 1024, "tokens": 512,
                                         "type": TYPE_HF_STELLA, "trustRemoteCode": True, "arch": _gte_arch()},
}


def find_model(model_name: str) -> Optional[dict]:
    """The registry entry of `model_name` (not a copy), or None: the one lookup over every table of served models."""
    for table in (MODELS, MPNET_MODELS, SIGLIP_MODELS, XLMR_MODELS, RESNET_MODELS, CONVNEXT_MODELS, BIG_VIT_MODELS,
                  EVA02_MODELS, GTE_MODELS):
        entry = table.get(model_name)
        if entry is not None:
            return entry
    return None


def all_models() -> Dict[str, dict]:
    """The served registry entries by name (a new dict over the same entries), except CONVNEXT_MODELS and
    BIG_VIT_MODELS.  The layer widths of these entries' towers are the served set the GEMM shape tests pin (384, 512,
    768, 1024), and their attention shapes the set the attention tests enumerate; the ConvNeXt CLIP text towers add
    width 640, and the big ViTs widths 1280 to 1664, padded head dims and 20 text heads, which
    tests/test_convnext_clip_gpu.py and tests/test_big_vit_gpu.py run instead.  EVA02_MODELS is in: its arch blocks
    keep the text tower (512 and 768 wide) at the top level, as the ResNet CLIP ones do, and its trunk in an "eva"
    block, whose layer shapes tests/test_eva02_kernels_gpu.py runs.  GTE_MODELS is in: its encoder is 1024 wide with a
    4096 hidden size, as the BERT-large models; its fused up | gate GEMM runs in tests/test_gte_kernels_gpu.py.
    served_models() has every served entry; find_model looks in every table."""
    return {**MODELS, **MPNET_MODELS, **SIGLIP_MODELS, **XLMR_MODELS, **RESNET_MODELS, **EVA02_MODELS, **GTE_MODELS}


def served_models() -> Dict[str, dict]:
    """Every served registry entry by name (a new dict over the same entries): all_models() and the tables it leaves
    out."""
    return {**all_models(), **CONVNEXT_MODELS, **BIG_VIT_MODELS}


def get_model_properties(model_name: str) -> dict:
    from .errors import UnknownModelError
    entry = find_model(model_name)
    if entry is None:
        raise UnknownModelError(f"Could not find model properties in model registry for model={model_name}. "
                                f"Model is not supported by default.")
    return copy.deepcopy(entry)
