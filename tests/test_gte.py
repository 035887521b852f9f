"""The Stella embedder (NewModel, the gte-v1.5 architecture) on the host: the registry entry vs the reference's, the
hf_stella loader type and its trustRemoteCode rule, the CPU oracle (tests/_gte_oracle.py) against transformers' Llama
rotary embedding and against a layer built from torch modules, and the WordPiece tokenizer the loader picks."""
import json
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import _gte_oracle as G
from marqo_b200 import model_registry as R

GOLDEN_DIR = Path(__file__).resolve().parent / "golden"


# ------------------------------------------------------------------------------------------------------------------
# Registry, model properties, loader
# ------------------------------------------------------------------------------------------------------------------
def test_entry_is_the_reference_entry():
    ref = json.loads((GOLDEN_DIR / "hf_registry_golden.json").read_text())[G.NAME]
    entry = R.GTE_MODELS[G.NAME]
    assert sorted(R.GTE_MODELS) == [G.NAME]
    assert {k: v for k, v in entry.items() if k not in ("arch", "type")} == {k: v for k, v in ref.items() if k != "type"}
    assert ref["type"] == "hf_stella" and entry["type"] == R.TYPE_HF_STELLA == "b200_hf_stella"
    assert entry["arch"] == G.engine_config(G.STELLA)
    assert R.find_model(G.NAME) is entry
    assert R.get_model_properties(G.NAME) == entry
    assert R.all_models()[G.NAME] is entry and R.served_models()[G.NAME] is entry
    assert entry["arch"]["width"] == entry["dimensions"]


def test_model_size_is_the_default():
    from marqo_b200 import s2_inference as s2
    assert s2._reference_type_name(R.TYPE_HF_STELLA) == "hf_stella"
    assert s2.get_model_size(G.NAME, R.get_model_properties(G.NAME)) == 0.66


def test_validate_model_properties_accepts_hf_stella():
    from marqo_b200 import s2_inference as s2
    by_name = s2.validate_model_properties(G.NAME, None)
    assert by_name["type"] == R.TYPE_HF_STELLA and by_name["tokens"] == 512
    custom = s2.validate_model_properties("my-stella", {"name": G.NAME, "type": "hf_stella", "dimensions": 1024,
                                                        "trustRemoteCode": True})
    assert custom["type"] == R.TYPE_HF_STELLA
    assert custom["tokens"] == 128      # hf's default
    assert custom["arch"] == R.GTE_MODELS[G.NAME]["arch"]


def test_loader_requires_trust_remote_code():
    """The reference's TestHuggingFaceStellaModel.test_trust_remote_code_validation against the hf_stella loader: absent
    or False is refused at construction with an error naming trustRemoteCode; True constructs."""
    from marqo_b200.errors import InvalidModelPropertiesError
    from marqo_b200.loaders import B200HuggingFace, get_model_loader
    loader = get_model_loader(G.NAME, {"type": R.TYPE_HF_STELLA})
    assert issubclass(loader, B200HuggingFace)
    for trust in (None, False):
        props = {k: v for k, v in {"name": "my_model", "type": "hf", "dimensions": 512,
                                   "trustRemoteCode": trust}.items() if v is not None}
        with pytest.raises(InvalidModelPropertiesError) as e:
            loader(device="cpu", model_properties=props)
        assert "trustRemoteCode" in str(e.value)
    assert loader(device="cpu", model_properties={"name": "my_model", "type": "hf", "dimensions": 512,
                                                  "trustRemoteCode": True}) is not None
    m = loader(device="cpu", model_properties=R.get_model_properties(G.NAME))
    assert m.max_seq_length == 512


def test_wordpiece_tokenizer_is_the_default(native_lib, tmp_path):
    """With a vocab.txt, the loader tokenizes with the C++ WordPiece tokenizer (uncased BERT): the same ids and mask as
    HF's BertWordPieceTokenizer on a small vocabulary, [CLS] first, [SEP] last, padded with 0."""
    from marqo_b200.loaders import LOADERS
    from marqo_b200.tokenizers import WordPieceTokenizer
    from oracle import tokenizers as OT
    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]", "what", "is", "the", "capital", "of", "france", "paris",
             "##is", "stella", "embed", "##ding", "##s", "?", ",", "."]
    path = tmp_path / "vocab.txt"
    path.write_text("\n".join(vocab) + "\n")
    m = LOADERS[R.TYPE_HF_STELLA](device="cpu", model_properties=dict(R.get_model_properties(G.NAME),
                                                                      vocab_file=str(path)))
    m.arch = m.model_properties["arch"]
    tok = m._default_tokenizer()
    assert isinstance(tok, WordPieceTokenizer)
    texts = ["What is the capital of France?", "Paris", "Stella embeddings, unknownword."]
    got = tok(texts, padding=True, truncation=True, max_length=512, return_tensors="np")
    ids, mask = OT.bert_encode_batch(OT.bert_wordpiece(vocab), texts, 512)
    np.testing.assert_array_equal(got["input_ids"], ids)
    np.testing.assert_array_equal(got["attention_mask"], mask)
    assert (got["input_ids"][:, 0] == vocab.index("[CLS]")).all()


# ------------------------------------------------------------------------------------------------------------------
# The oracle
# ------------------------------------------------------------------------------------------------------------------
def test_inv_freq_is_the_ntk_formula():
    f = G.inv_freq(G.STELLA)
    assert f[0] == pytest.approx(2.0 ** (-1 / 32))
    assert f[31] == pytest.approx(320000.0 ** (-62 / 64) * 2.0 ** (-1 / 32))
    # factor 1 is the unscaled RotaryEmbedding: base^(-2j/64)
    plain = G.inv_freq(G.GteCfg(rope_ntk_factor=1.0))
    torch.testing.assert_close(plain, 160000.0 ** (-2.0 * torch.arange(32, dtype=torch.float64) / 64))


def test_rotation_matches_llama_apply_rotary_pos_emb():
    """The oracle's rotate-half against transformers' Llama apply_rotary_pos_emb with the same angles."""
    from transformers.models.llama.modeling_llama import apply_rotary_pos_emb
    g = torch.Generator().manual_seed(3)
    B, S, H = 2, 77, 4
    q, k = torch.randn(B, S, H, 64, generator=g), torch.randn(B, S, H, 64, generator=g)
    th = G.rope_angles(G.STELLA, S)
    cos, sin = th.cos().float(), th.sin().float()
    emb_cos, emb_sin = torch.cat([cos, cos], -1), torch.cat([sin, sin], -1)     # [S, 64], as RotaryEmbedding caches
    rq, rk = apply_rotary_pos_emb(q.transpose(1, 2), k.transpose(1, 2), emb_cos[None], emb_sin[None])
    torch.testing.assert_close(G.rotate(q, cos, sin), rq.transpose(1, 2), rtol=0, atol=1e-6)
    torch.testing.assert_close(G.rotate(k, cos, sin), rk.transpose(1, 2), rtol=0, atol=1e-6)


def _module_layer(sd, p, cfg, x, keep, cos, sin):
    """NewLayer from torch.nn modules and F.scaled_dot_product_attention with the key mask."""
    w, H, mlp = cfg.width, cfg.heads, cfg.mlp

    def linear(name, n_out, n_in, bias=True):
        lin = torch.nn.Linear(n_in, n_out, bias=bias)
        lin.weight.data.copy_(sd[p + name + ".weight"])
        if bias:
            lin.bias.data.copy_(sd[p + name + ".bias"])
        return lin

    def norm(name):
        ln = torch.nn.LayerNorm(w, eps=cfg.ln_eps)
        ln.weight.data.copy_(sd[p + name + ".weight"])
        ln.bias.data.copy_(sd[p + name + ".bias"])
        return ln

    B, S, _ = x.shape
    q, k, v = linear("attention.qkv_proj", 3 * w, w)(x).chunk(3, dim=-1)
    heads = lambda t: t.view(B, S, H, 64).transpose(1, 2)                   # noqa: E731
    c, s = torch.cat([cos, cos], -1), torch.cat([sin, sin], -1)

    def rot(t):
        half = torch.cat([-t[..., 32:], t[..., :32]], dim=-1)               # rotate_half
        return t * c + half * s

    o = F.scaled_dot_product_attention(rot(heads(q)), rot(heads(k)), heads(v), attn_mask=keep[:, None, None, :])
    x = norm("attn_ln")(x + linear("attention.o_proj", w, w)(o.transpose(1, 2).reshape(B, S, w)))
    up, gate = torch.split(linear("mlp.up_gate_proj", 2 * mlp, w, bias=False)(x), mlp, dim=-1)
    return norm("mlp_ln")(x + linear("mlp.down_proj", w, mlp)(F.gelu(gate) * up))


@torch.no_grad()
def test_oracle_layer_matches_torch_modules():
    cfg = G.GteCfg(width=256, layers=1, heads=4, mlp=512, vocab=500)
    sd = G.make_gte_weights(cfg, seed=8)
    g = torch.Generator().manual_seed(9)
    B, S = 3, 40
    x = torch.randn(B, S, cfg.width, generator=g)
    keep = torch.ones(B, S, dtype=torch.bool)
    keep[1, 17:] = False
    keep[2, 1:] = False
    th = G.rope_angles(cfg, S)
    cos, sin = th.cos().float(), th.sin().float()
    got = G.layer(sd, "encoder.layer.0.", cfg, x, keep, cos, sin)
    want = _module_layer(sd, "encoder.layer.0.", cfg, x, keep, cos, sin)
    torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-4)


def test_oracle_pooling_ignores_padding():
    """Padding a batch further changes no row: the keys are masked and the mean counts the real tokens only."""
    cfg = G.tiny_gte()
    sd = G.make_gte_weights(cfg, seed=4)
    ids, mask = G.ragged_ids(torch.Generator().manual_seed(1), [1, 9, 30], 30, cfg.vocab)
    a = G.gte_encode(sd, cfg, ids, mask)
    wide = torch.zeros(3, 45, dtype=torch.long)
    wide_mask = torch.zeros(3, 45, dtype=torch.long)
    wide[:, :30], wide_mask[:, :30] = ids, mask
    torch.testing.assert_close(G.gte_encode(sd, cfg, wide, wide_mask), a, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(a.norm(dim=1), torch.ones(3))
