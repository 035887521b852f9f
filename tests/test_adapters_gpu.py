"""GPU tests of the reference-facing adapters: vectorise() through the loader classes (B1) and the VespaClient-shaped
GpuTensorIndex (B2), against the oracle."""
import numpy as np
import pytest
import torch

import _checks as K
from oracle import encoders as E

pytestmark = pytest.mark.gpu

TINY_BERT_ARCH = dict(width=128, layers=2, heads=2, mlp=512, vocab=1000, max_pos=64, type_vocab=2, pool="mean")
TINY_CLIP_ARCH = dict(embed_dim=128, act="gelu", mean=E.OPENAI_CLIP_MEAN, std=E.OPENAI_CLIP_STD,
                      vision=dict(width=128, layers=2, heads=2, mlp=512, patch=32, image_size=224),
                      text=dict(width=128, layers=2, heads=2, mlp=512, ctx=77, vocab=1000))


def test_vectorise_hf_loader_end_to_end(gpu_required, monkeypatch):
    from marqo_b200 import s2_inference as s2, weights as Wt
    s2.clear_loaded_models()
    tok = K.WordTokenizer(2, 3, 5)
    props = {"name": "tiny-bert", "dimensions": 128, "type": "hf", "tokens": 32, "arch": TINY_BERT_ARCH,
             "random_init": 77, "tokenizer": tok}
    rng = np.random.default_rng(0)
    sentences = [" ".join(f"w{int(x)}" for x in rng.integers(0, 990, size=n)) for n in rng.integers(1, 45, size=21)]
    monkeypatch.setenv("MARQO_MAX_VECTORISE_BATCH_SIZE", "8")           # 3 sub-batches, each padded to its own longest
    out = s2.vectorise("tiny-bert", sentences, model_properties=props, device="cuda:0", normalize_embeddings=True)
    assert isinstance(out, list) and len(out) == 21 and len(out[0]) == 128 and isinstance(out[0][0], float)
    sd = {k: torch.from_numpy(v) for k, v in Wt.random_bert_weights(TINY_BERT_ARCH, 77).items()}
    cfg = E.BertCfg(128, 2, 2, 512, vocab=1000, max_pos=64)
    ref = []
    for i in range(0, 21, 8):                                            # the reference pads per sub-batch (Appendix A)
        t = tok(sentences[i:i + 8], max_length=32)
        ref.append(E.bert_encode(sd, cfg, torch.from_numpy(t["input_ids"]), torch.from_numpy(t["attention_mask"])))
    K.assert_embeddings_match(out, torch.cat(ref))
    one = s2.vectorise("tiny-bert", sentences[3], model_properties=props, device="cuda:0")
    K.assert_embeddings_match(one, torch.cat(ref)[3:4], unit_norm=False)   # str == [str] (test_encoding.py:28-60)
    assert len(s2._available_models) == 1
    s2.eject_model("tiny-bert", "cuda:0", props)
    assert len(s2._available_models) == 0


def test_vectorise_clip_loader_images_and_text(gpu_required, monkeypatch):
    from PIL import Image
    from marqo_b200 import s2_inference as s2, weights as Wt
    s2.clear_loaded_models()
    ids_table = {}

    def clip_tok(texts):
        out = np.zeros((len(texts), 77), np.int64)
        for i, t in enumerate(texts):
            w = [int(x) for x in t.split()]
            out[i, 0] = 998
            out[i, 1:1 + len(w)] = w
            out[i, 1 + len(w)] = 999
        return out

    props = {"name": "tiny-clip", "dimensions": 128, "type": "open_clip", "arch": TINY_CLIP_ARCH, "random_init": 5,
             "tokenizer": clip_tok, "max_batch": 8}
    rng = np.random.default_rng(1)
    raw = [rng.integers(0, 256, size=(224, 224, 3), dtype=np.uint8) for _ in range(5)]
    raw.append(rng.integers(0, 256, size=(260, 330, 3), dtype=np.uint8))        # one odd-sized image: resize path
    pil = [Image.fromarray(a) for a in raw]
    sd = {k: torch.from_numpy(v) for k, v in Wt.random_clip_weights(TINY_CLIP_ARCH, 5).items()}
    cfg = E.tiny_clip()
    ref = E.clip_encode_image(sd, cfg, torch.stack([E.clip_preprocess_pil(p) for p in pil]))
    monkeypatch.setenv("MARQO_MAX_VECTORISE_BATCH_SIZE", "4")
    out = s2.vectorise("tiny-clip", pil, model_properties=props, device="cuda:0", modality=s2.Modality.IMAGE)
    K.assert_embeddings_match(out, ref, unit_norm=False)
    # what the download threads hand over: model.preprocess(pil) tensors (add_docs.py:129-134)
    key = next(iter(s2._available_models))
    model = s2._available_models[key]["model"]
    pre = [model.preprocess(p) for p in pil]
    assert pre[0].dtype == torch.uint8 and tuple(pre[0].shape) == (224, 224, 3)
    out2 = s2.vectorise("tiny-clip", pre, model_properties=props, device="cuda:0", modality=s2.Modality.IMAGE)
    assert out2 == out
    # already-preprocessed float CHW tensors pass through unchanged (abstract_clip_model.py:108-111)
    chw = [E.clip_preprocess_pil(p) for p in pil[:3]]
    got = s2.vectorise("tiny-clip", chw, model_properties=props, device="cuda:0", modality=s2.Modality.IMAGE)
    K.assert_embeddings_match(got, ref[:3], unit_norm=False)
    # text
    texts = ["1 2 3", "7", " ".join(str(i) for i in range(10, 60))]
    tref = E.clip_encode_text(sd, cfg, torch.from_numpy(clip_tok(texts)))
    got = s2.vectorise("tiny-clip", texts, model_properties=props, device="cuda:0")
    K.assert_embeddings_match(got, tref, unit_norm=False)
    assert np.array_equal(model.encode_text(texts), model.encode(texts))         # test_encoding.py:334-370
    s2.clear_loaded_models()


def test_vectorise_with_cxx_tokenizers(gpu_required, tmp_path):
    """f2 end to end: model_properties point at vocabulary FILES; strings go through the C++ tokenizers and the CUDA
    encoders; the expectation tokenises with the oracle tokenizers (HF `tokenizers` / restated SimpleTokenizer)."""
    from marqo_b200 import s2_inference as s2, weights as Wt
    from oracle import tokenizers as OT
    s2.clear_loaded_models()
    # ---- BERT + WordPiece
    words = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + [f"w{i}" for i in range(600)] + \
            ["##ing", "##s", "##ed", ",", ".", "!", "caf", "##e", "cafe"]
    vocab_file = tmp_path / "vocab.txt"
    vocab_file.write_text("\n".join(words) + "\n", encoding="utf-8")
    props = {"name": "tiny-bert-wp", "dimensions": 128, "type": "hf", "tokens": 32, "arch": TINY_BERT_ARCH,
             "random_init": 77, "vocab_file": str(vocab_file)}
    sentences = ["w1 w2 w3ing, w4s!", "Café W5 w599ed unknownword.", "w7", "w8 " * 60]
    out = s2.vectorise("tiny-bert-wp", sentences, model_properties=props, device="cuda:0", normalize_embeddings=True)
    ids, mask = OT.bert_encode_batch(OT.bert_wordpiece(words), sentences, 32)
    sd = {k: torch.from_numpy(v) for k, v in Wt.random_bert_weights(TINY_BERT_ARCH, 77).items()}
    ref = E.bert_encode(sd, E.BertCfg(128, 2, 2, 512, vocab=1000, max_pos=64), torch.from_numpy(ids), torch.from_numpy(mask))
    K.assert_embeddings_match(out, ref, unit_norm=False)
    # ---- CLIP text tower + byte-level BPE
    corpus = ["a photo of a cat", "a photo of a dog", "the quick brown fox", "hello world, it's me"] * 2
    merges = OT.train_toy_merges(corpus, 300)
    merges_file = tmp_path / "bpe.txt"
    merges_file.write_text(merges, encoding="utf-8")
    cprops = {"name": "open_clip/tiny/test", "dimensions": 128, "type": "open_clip", "arch": TINY_CLIP_ARCH,
              "random_init": 5, "merges_file": str(merges_file)}
    texts = ["A photo of a CAT", "hello &amp; world", "the quick brown dog's photo " * 20]
    got = s2.vectorise("open_clip/tiny/test", texts, model_properties=cprops, device="cuda:0")
    tok_ids = OT.SimpleTokenizerOracle(merges)(texts)
    assert tok_ids.max() < TINY_CLIP_ARCH["text"]["vocab"]
    csd = {k: torch.from_numpy(v) for k, v in Wt.random_clip_weights(TINY_CLIP_ARCH, 5).items()}
    s2.clear_loaded_models()
    K.assert_embeddings_match(got, E.clip_encode_text(csd, E.tiny_clip(), torch.from_numpy(tok_ids)), unit_norm=False)


def _doc(doc_id, fields, embs):
    f = dict(fields)
    for name, (chunks, vecs) in embs.items():
        f[f"marqo__chunks_{name}"] = chunks
        f[f"marqo__embeddings_{name}"] = {str(i): v.tolist() for i, v in enumerate(vecs)}
    return {"id": doc_id, "fields": f}


def _yql(schema, fields, k):
    terms = " OR ".join(f"({{targetHits:{k}, approximate:False, hnsw.exploreAdditionalHits:0}}"
                        f"nearestNeighbor(marqo__embeddings_{f}, marqo__query_embedding))" for f in fields)
    return f"select * from {schema} where ({terms})"


def test_gpu_tensor_index_feed_query_highlights_overwrite_delete(gpu_required):
    from _filter_scenario import run_feed_query_scenario
    run_feed_query_scenario()


def test_gpu_tensor_index_score_modifiers(gpu_required):
    """Tensor search with score_modifiers (tensor_search.py -> vespa_index.py:106-150): the query carries
    marqo__mult_weights_tensor / marqo__add_weights_tensor, documents carry marqo__score_modifiers."""
    from _filter_scenario import run_score_modifier_scenario
    run_score_modifier_scenario()


def test_gpu_tensor_index_snapshot_restart(gpu_required, tmp_path):
    """f4 corpus persistence: save -> load on a fresh object gives the same hits, highlights, modifiers, get_batch."""
    from marqo_b200.gpu_tensor_index import GpuTensorIndex, gather_documents_from_response
    rng = np.random.default_rng(21)
    D = 64

    def unit(m):
        x = rng.standard_normal((m, D)).astype(np.float32)
        return x / np.linalg.norm(x, axis=1, keepdims=True)

    ix = GpuTensorIndex()
    docs = [_doc(f"d{i}", {"marqo__id": f"d{i}", "n": i, "marqo__score_modifiers": {"pop": float(i % 5 + 1)}},
                 {"title": ([f"t{i}"], unit(1)), "body": ([f"b{i}.{j}" for j in range(2)], unit(2))}) for i in range(30)]
    ix.feed_batch(docs, "s1")
    ix.delete_batch(["d4"], "s1")
    ix.feed_batch([_doc("d9", {"marqo__id": "d9", "n": 900}, {"title": (["new"], unit(1))})], "s1")   # overwrite
    q = unit(1)[0]
    plain = {"marqo__query_embedding": q.tolist()}
    mod = dict(plain, marqo__mult_weights_tensor={"pop": 0.7}, marqo__add_weights_tensor={"pop": 0.01})
    before = [ix.query(_yql("s1", ["title", "body"], 8), hits=8, ranking="embedding_similarity", model_restrict="s1",
                       query_features=f) for f in (plain, mod)]
    ix.save(str(tmp_path / "snap"))
    ix.close()
    again = GpuTensorIndex.load(str(tmp_path / "snap"))
    after = [again.query(_yql("s1", ["title", "body"], 8), hits=8, ranking="embedding_similarity", model_restrict="s1",
                         query_features=f) for f in (plain, mod)]
    for b, a in zip(before, after):
        assert [h.id for h in b.hits] == [h.id for h in a.hits]
        assert [h.relevance for h in b.hits] == [h.relevance for h in a.hits]
        assert gather_documents_from_response(b) == gather_documents_from_response(a)
    assert again.get_document_count("s1") == 29
    got = again.get_batch(["d9", "d4"], "s1")
    assert got.responses[0].status == 200 and got.responses[0].document.fields["n"] == 900
    assert got.responses[1].status == 404
    # the restored index keeps accepting documents
    assert not again.feed_batch([_doc("fresh", {"marqo__id": "fresh"}, {"title": (["x"], unit(1))})], "s1").errors
    assert again.get_document_count("s1") == 30
    again.close()


def test_gpu_tensor_index_filtered_search(gpu_required):
    """Tensor search with a filter (tensor_search.py -> unstructured_vespa_index.py:59-66,135-226): exact top-k among
    the documents the filter keeps; scenario shared with the CPU stand-in run (tests/_filter_scenario.py)."""
    from _filter_scenario import run_filtered_search_scenario
    run_filtered_search_scenario()


def test_concurrent_encode_calls_are_serialised_per_handle(gpu_required):
    """Marqo calls encode() from up to 16 request threads with no lock (SURVEY §8b); the handle serialises internally."""
    import threading
    from marqo_b200 import weights as Wt
    from marqo_b200.engine import Encoder
    enc = Encoder("bert", TINY_BERT_ARCH, Wt.random_bert_weights(TINY_BERT_ARCH, 3), max_batch=16)
    rng = np.random.default_rng(0)
    inputs = [rng.integers(1, 999, size=(int(rng.integers(1, 12)), int(rng.integers(2, 60)))).astype(np.int32) for _ in range(24)]
    serial = [enc.encode_tokens(x) for x in inputs]
    out = [None] * len(inputs)

    def work(lo):
        for i in range(lo, len(inputs), 6):
            out[i] = enc.encode_tokens(inputs[i])

    threads = [threading.Thread(target=work, args=(k,)) for k in range(6)]
    [t.start() for t in threads]
    [t.join() for t in threads]
    for a, b in zip(serial, out):
        np.testing.assert_array_equal(a, b)          # same kernels, same order of arithmetic -> bitwise equal
    enc.close()


def test_vectorise_decodes_jpegs_on_the_gpu(gpu_required, monkeypatch):
    """The ingest seam end to end: lazy PIL images (Image.open, image_download.py:146-152) -> model.preprocess hands the
    still-encoded JPEG over -> vectorise() -> encode_image decodes the batch on the GPU (bit-exact with Pillow), resizes
    and encodes.  Same vectors as handing over Pillow-decoded pixels; a progressive file rides along through Pillow."""
    import io
    from PIL import Image
    from marqo_b200 import s2_inference as S2
    from marqo_b200.image_decode import EncodedImage
    rng = np.random.default_rng(4)
    files = []
    for i, (h, w) in enumerate([(300, 400), (224, 224), (500, 333), (300, 400)]):
        img = Image.fromarray(np.kron(rng.integers(0, 256, size=(h // 20 + 1, w // 20 + 1, 3), dtype=np.uint8),
                                      np.ones((20, 20, 1), np.uint8))[:h, :w])
        b = io.BytesIO()
        img.save(b, format="JPEG", quality=85, subsampling=(0, 1, 2, 2)[i], progressive=(i == 3))
        files.append(b.getvalue())
    props = {"name": "tiny-clip", "dimensions": 128, "type": "open_clip", "arch": TINY_CLIP_ARCH, "random_init": 5,
             "max_batch": 8}
    S2.clear_loaded_models()
    pre = S2.load_multimodal_model_and_get_preprocessors("tiny-clip", props, device="cuda:0")[1]["image"]
    media = [pre(Image.open(io.BytesIO(f))).to("cuda:0") for f in files]
    assert all(isinstance(m, EncodedImage) for m in media[:3])
    got = np.asarray(S2.vectorise("tiny-clip", media, model_properties=props, device="cuda:0", normalize_embeddings=True,
                                  modality=S2.Modality.IMAGE))
    decoded = [np.asarray(Image.open(io.BytesIO(f)).convert("RGB")) for f in files]
    want = np.asarray(S2.vectorise("tiny-clip", [torch.from_numpy(d) for d in decoded], model_properties=props,
                                   device="cuda:0", normalize_embeddings=True, modality=S2.Modality.IMAGE))
    np.testing.assert_array_equal(got, want)          # identical pixels -> identical kernels -> identical vectors
    S2.clear_loaded_models()
