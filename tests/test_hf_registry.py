"""The engine's hf/* registry entries vs the reference's own (tests/golden/hf_registry_golden.json, written by
tests/golden/make_hf_registry_golden.py), their `arch` shapes vs what the kernels serve, and the CPU oracle's BERT vs
transformers.BertModel at the head_dim-32 shapes of the 384-wide embedders."""
import json
from pathlib import Path

import pytest
import torch

from marqo_b200 import model_registry as R
from oracle import encoders as E

GOLDEN = Path(__file__).resolve().parent / "golden" / "hf_registry_golden.json"
HF = {k: v for k, v in R.MODELS.items() if k.startswith("hf/")}

MINILM_L6 = E.BertCfg(384, 6, 12, 1536)
E5_SMALL = E.BertCfg(384, 12, 12, 1536)


def test_every_hf_entry_is_the_reference_entry():
    ref = json.loads(GOLDEN.read_text())
    assert len(HF) == 18
    for name, entry in HF.items():
        assert name in ref, name
        want = dict(ref[name], type=R.TYPE_HF)
        got = {k: v for k, v in entry.items() if k != "arch"}
        assert got == want, name
        assert R.get_model_properties(name) == entry


def test_small_bert_entries():
    for name in ("hf/all-MiniLM-L6-v1", "hf/all-MiniLM-L6-v2", "hf/all_datasets_v3_MiniLM-L6",
                 "hf/all_datasets_v4_MiniLM-L6"):
        a = HF[name]["arch"]
        assert (a["width"], a["layers"], a["heads"], a["mlp"]) == (384, 6, 12, 1536), name
    for name in ("hf/all_datasets_v3_MiniLM-L12", "hf/all_datasets_v4_MiniLM-L12", "hf/e5-small", "hf/e5-small-v2",
                 "hf/e5-small-unsupervised", "hf/bge-small-en-v1.5"):
        a = HF[name]["arch"]
        assert (a["width"], a["layers"], a["heads"], a["mlp"]) == (384, 12, 12, 1536), name
    # head count does not change a weight shape: e5-small-v2 with 6 heads would load a real checkpoint and be wrong
    assert HF["hf/e5-small-v2"]["arch"]["heads"] == 12
    assert HF["hf/e5-large"]["tokens"] == 192 and HF["hf/e5-large"]["model_size"] == 1.3
    assert HF["hf/e5-base"]["tokens"] == 192


@pytest.mark.parametrize("name", sorted(HF))
def test_arch_is_servable(name):
    a = HF[name]["arch"]
    assert a["width"] % a["heads"] == 0 and a["width"] // a["heads"] in (32, 64)
    assert a["width"] % 128 == 0 and a["mlp"] % 64 == 0
    assert (a["vocab"], a["max_pos"], a["type_vocab"], a["pool"]) == (30522, 512, 2, "mean")
    assert HF[name]["dimensions"] == a["width"]


@pytest.mark.parametrize("cfg", [MINILM_L6, E5_SMALL], ids=["minilm_l6", "e5_small"])
def test_bert_head_dim_32_matches_hf(cfg):
    """The oracle's BERT restatement (oracle/encoders.py) vs transformers.BertModel at head_dim 32, mean pooling."""
    from transformers import BertConfig, BertModel
    sd = E.make_bert_weights(cfg, seed=21)
    hc = BertConfig(vocab_size=cfg.vocab, hidden_size=cfg.width, num_hidden_layers=cfg.layers,
                    num_attention_heads=cfg.heads, intermediate_size=cfg.mlp, max_position_embeddings=cfg.max_pos,
                    type_vocab_size=cfg.type_vocab, hidden_act="gelu", layer_norm_eps=cfg.ln_eps,
                    hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, attn_implementation="eager")
    m = BertModel(hc, add_pooling_layer=False).eval()
    missing = m.load_state_dict(sd, strict=False)
    assert not missing.unexpected_keys and all("position_ids" in k for k in missing.missing_keys)
    g = torch.Generator().manual_seed(4)
    ids = torch.randint(1000, 30000, (4, 40), generator=g)
    mask = torch.ones(4, 40, dtype=torch.long)
    for b, L in enumerate([40, 12, 1, 27]):
        mask[b, L:] = 0
        ids[b, L:] = 0
    with torch.no_grad():
        out = m(input_ids=ids, attention_mask=mask)
    last = out.last_hidden_state.masked_fill(~mask[..., None].bool(), 0.0)
    ref = torch.nn.functional.normalize(last.sum(dim=1) / mask.sum(dim=1)[..., None], p=2, dim=1)
    got = E.bert_encode(sd, cfg, ids, mask, normalize=True)
    torch.testing.assert_close(got, ref, rtol=1e-4, atol=1e-4)
