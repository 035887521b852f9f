/* marqo_b200 — C ABI of the H100-native (sm_90a) embed-and-score engine.
 *
 * The reference (marqo-ai/marqo) has NO foreign-function interface on this path: it calls
 * open_clip / transformers / torch for the encoders and an HTTP POST to Vespa for the score
 * step.  This header is therefore the boundary a Marqo maintainer would bind from Python
 * (ctypes — see INTEGRATION.md) underneath the reference's two pure-Python seams:
 *
 *   B1  encoder seam   model.encode(...) objects held by s2_inference._available_models
 *                      (src/marqo/s2_inference/s2_inference.py:123-158, :520-568;
 *                       loaders map src/marqo/s2_inference/model_registry.py:2133-2145)
 *   B2  score seam     VespaClient.query()/feed_batch()
 *                      (src/marqo/vespa/vespa_client.py:198-242, :267-296), consumed at
 *                      src/marqo/tensor_search/tensor_search.py:2189 and
 *                      src/marqo/core/vespa_index/add_documents_handler.py:177
 *
 * Conventions: plain C, opaque handles, caller-owned host buffers, every function returns an
 * int status (B200_OK == 0) and leaves a thread-local message readable through
 * b200_last_error().  Handles are internally serialised (one mutex + one CUDA stream per
 * handle), so concurrent calls from Marqo's request threadpool are safe.  There is no CPU
 * fallback: without a usable sm_90 device every compute entry point fails with
 * B200_ERR_NO_DEVICE.
 */
#ifndef MARQO_B200_H
#define MARQO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_ABI_VERSION 1

enum b200_status {
    B200_OK = 0,
    B200_ERR_INVALID_ARG = 1,
    B200_ERR_NO_DEVICE = 2,
    B200_ERR_CUDA = 3,
    B200_ERR_OOM = 4,
    B200_ERR_UNSUPPORTED = 5,
    B200_ERR_INTERNAL = 6,
    B200_ERR_MISSING_WEIGHT = 7
};

int b200_abi_version(void);
/* Thread-local text of the last failure on this thread ("" if none). */
const char* b200_last_error(void);
/* Number of visible CUDA devices with compute capability 10.x. */
int b200_device_count(int* out_count);

/* Page-locked host memory (cudaHostAlloc, portable) for staging inputs: host-to-device copies from it run at the full
 * PCIe rate.  The reference stages every image separately (`.to(device)` per image at
 * src/marqo/tensor_search/add_docs.py:129-134); the adapters assemble a batch in one such buffer instead. */
int b200_host_alloc(size_t bytes, void** out);
int b200_host_free(void* p);

/* ===================================================================================== */
/* Score + top-k over a GPU-resident embedding matrix  (SURVEY §8 a8; replaces the Vespa   */
/* nearestNeighbor / closeness / top-k round trip specified by                            */
/* src/marqo/core/unstructured_vespa_index/unstructured_vespa_index.py:59-133,            */
/* src/marqo/core/structured_vespa_index/structured_vespa_index.py:403-446,645-688 and    */
/* src/marqo/core/unstructured_vespa_index/unstructured_vespa_schema.py:155-166,225-230). */
/* ===================================================================================== */

typedef struct b200_index b200_index;

/* Distance metrics: names from src/marqo/core/models/marqo_index.py:63-69. */
enum b200_metric {
    B200_METRIC_PRENORMALIZED_ANGULAR = 0, /* distance = 1 - q.e           closeness = 1/(1+d) */
    B200_METRIC_ANGULAR = 1,               /* distance = acos(cos(q,e))    closeness = 1/(1+d) */
    B200_METRIC_DOTPRODUCT = 2,            /* distance = -q.e              closeness = q.e (raw) */
    B200_METRIC_EUCLIDEAN = 3              /* distance = |q-e|             closeness = 1/(1+d)  (scan key 2 q.e - |e|^2) */
};

/* Create an empty row store of fp16[capacity_rows, dim] on `device` (grows on demand).
 * dim must be a multiple of 64 and <= 4096; any other dim returns B200_ERR_INVALID_ARG.  Up to 1024 the scan keeps the
 * query block resident in shared memory; above it the query block is streamed beside the corpus. */
int b200_index_create(int device, int dim, int metric, int64_t capacity_rows, b200_index** out);
int b200_index_destroy(b200_index* ix);

/* Append m chunk embeddings (fp32, host, row-major [m, dim]).  doc_ids[i] is the internal
 * document number (>= 0) the chunk belongs to; NULL means "one chunk per document, document
 * number == row number".  Rows of one document need not be contiguous.  Replaces
 * VespaClient.feed_batch for the tensor fields (vespa_client.py:267-296; the per-document
 * {"<chunk>": [floats]} blocks built at
 * src/marqo/core/semi_structured_vespa_index/semi_structured_document.py:127-143). */
int b200_index_add(b200_index* ix, const float* vecs, const int32_t* doc_ids, int64_t m);
/* Same, source already on the index's device (fp32 [m, dim]); used by the add_documents fast
 * path that never materialises List[List[float]] on the host. */
int b200_index_add_device(b200_index* ix, const float* d_vecs, const int32_t* d_doc_ids, int64_t m);
/* Same with the embeddings on the device (straight out of b200_model_encode_*_device) and the document numbers on the
 * host: the add_documents fast path — vectors never visit the host, the small id list does not need a device buffer
 * of the caller's (core/vespa_index/add_documents_handler.py:160-177 feeds what
 * core/inference/tensor_fields_container.py:196-223 collected). */
int b200_index_add_device_docs(b200_index* ix, const float* d_vecs, const int32_t* doc_ids, int64_t m);
/* Rows whose values are not finite or do not fit the fp16 row store (|x| > 65504 after the angular metric's
 * normalisation) are rejected by all three add calls with B200_ERR_INVALID_ARG; nothing of the batch is kept. */
/* Tombstone every row of a document (add_documents replaces by _id:
 * src/marqo/core/vespa_index/add_documents_handler.py:140,258).  O(rows): prefer b200_index_delete_rows when the
 * caller knows the document's rows. */
int b200_index_delete_doc(b200_index* ix, int32_t doc_id);
/* Tombstone the listed rows (the adapter keeps document -> rows): one small scatter per batch of replaced / deleted
 * documents instead of a corpus-wide pass per document. */
int b200_index_delete_rows(b200_index* ix, const int32_t* rows, int64_t n);
/* Squeeze tombstoned rows out of the matrix.  out_new_of_old: caller buffer of (current) num_rows int32 — the new row
 * number of every old row, -1 for a dead one; *out_rows = rows left.  Row numbers returned by earlier searches are
 * invalid afterwards. */
int b200_index_compact(b200_index* ix, int32_t* out_new_of_old, int64_t* out_rows);
int b200_index_num_rows(b200_index* ix, int64_t* out_rows);
int b200_index_info(b200_index* ix, int* out_dim, int* out_metric, int* out_device);
/* Copy row `row` back as fp32 (get_batch / use_existing_tensors:
 * add_documents_handler.py:160-165). */
int b200_index_get_row(b200_index* ix, int64_t row, float* out_vec);
int b200_index_get_rows(b200_index* ix, const int64_t* rows, int64_t n, float* out_vecs);

/* Exact search.  q: fp32 host [nq, dim].  For every query returns the k best DOCUMENTS under
 *   score(doc) = max over the document's live rows of closeness(q, row)
 * ordered by (score desc, doc_id asc).  out_doc/out_row/out_score are [nq, k]; unused slots are
 * filled with doc = row = -1, score = -inf.  out_row is the arg-max chunk row (Vespa's
 * closest(), used for _highlights: structured_vespa_index.py:942-1000).  out_score is the
 * closeness ("relevance", tensor_search.py:1771-1791) computed in fp64 from an exactly
 * rescored dot product. */
int b200_index_search(b200_index* ix, const float* q, int nq, int k, int32_t* out_doc, int32_t* out_row,
                      double* out_score);
/* How exactness is guaranteed (score.cu header): the tensor-core pass only SELECTS candidates, which are re-scored in
 * fp64; a per-query guard proves that no row outside the candidate set can reach the k-th exact score, and queries
 * that fail it (exact ties / near-ties across the candidate boundary, k beyond the per-SM lists) are answered by a
 * second threshold-collect pass over the corpus.  k <= 160 is normally ONE pass; any k <= 11000 is supported
 * (limit <= 1000 and offset <= 10000: src/marqo/api/configs.py:24-25). */
/* Same with queries and outputs resident on the index's device; asynchronous on the handle's
 * stream unless sync != 0.  With sync == 0 one fallback pass is enqueued unconditionally (it exits at once when no
 * query needs it); a query that would need MORE than one fallback pass cannot be driven from the host then —
 * b200_index_search_stats reports how often that happened (out_unresolved; 0 in every test and benchmark). */
int b200_index_search_device(b200_index* ix, const float* d_q, int nq, int k, int32_t* d_out_doc,
                             int32_t* d_out_row, double* d_out_score, int sync);
/* Counters since creation: groups of <= 64 queries searched, queries that failed the guard, fallback passes run by
 * the synchronous entry points, groups the asynchronous entry point left unresolved.  Any pointer may be NULL. */
int b200_index_search_stats(b200_index* ix, int64_t* out_groups, int64_t* out_flagged, int64_t* out_collect_passes,
                            int64_t* out_unresolved);

/* Search options: score modifiers (below) and a document FILTER.  filter_bits is a host bitset over LOCAL document
 * numbers (bit d of word d/32 set = document d may match; documents >= filter_docs are excluded): the adapter compiles
 * the ` AND <filter>` text Marqo appends to a tensor query (unstructured_vespa_index.py:59-66,135-226;
 * structured_vespa_index.py:690-793) to this bitset once per distinct filter string and the scan applies it where it
 * reads the row -> document map, next to the tombstone check — a filtered query costs one pass, whatever its
 * selectivity.  filter_tag != 0 names the bitset: the device copy is reused while tag and filter_docs repeat. */
typedef struct b200_search_opts {
    const int32_t* mult_cols;
    const double* mult_w;
    int32_t n_mult;
    const int32_t* add_cols;
    const double* add_w;
    int32_t n_add;
    const uint32_t* filter_bits;
    int64_t filter_docs;
    uint64_t filter_tag;
} b200_search_opts;
/* b200_index_search with options (opts == NULL: plain search). */
int b200_index_search_ex(b200_index* ix, const float* q, int nq, int k, const b200_search_opts* opts, int32_t* out_doc,
                         int32_t* out_row, double* out_score);

/* Score modifiers (SURVEY §8 f3).  Per-document numeric attributes: the `marqo__score_modifiers`
 * tensor<double>(p{}) field every document is fed with
 * (src/marqo/core/unstructured_vespa_index/unstructured_document.py:25,110-125;
 * src/marqo/core/semi_structured_vespa_index/semi_structured_document.py:23,104-117).  The host maps each
 * attribute NAME to a column number in [0, B200_MAX_ATTRIBUTE_COLUMNS).  values == NULL removes the cells (the
 * document no longer has the attribute); column == -1 with values == NULL removes the documents' cells in every
 * column (document overwritten or deleted).  Document numbers are LOCAL (before b200_index_set_doc_offset). */
#define B200_MAX_ATTRIBUTE_COLUMNS 64
int b200_index_set_attributes(b200_index* ix, int column, const int32_t* doc_ids, const double* values, int64_t n);
/* Many (column, document, value) cells in one call — one feed_batch, one launch. */
int b200_index_set_attributes_multi(b200_index* ix, const int32_t* columns, const int32_t* doc_ids, const double* values,
                                    int64_t n);
/* b200_index_search with the rank-profile function
 *   modify(score, mult_weights, add_weights) =
 *       if(count(mult_weights * attr) == 0, 1, reduce(mult_weights * attr, prod)) * score + reduce(add_weights * attr, sum)
 * (src/marqo/core/unstructured_vespa_index/unstructured_vespa_schema.py:266-271, applied at :225-230) evaluated
 * inside the scan, before top-k; `score` = closeness of the document's best chunk.  The sparse products run over the
 * attribute cells a document has.  mult_cols/mult_w and add_cols/add_w are the query tensors
 * `marqo__mult_weights_tensor` / `marqo__add_weights_tensor` (src/marqo/core/vespa_index/vespa_index.py:124-150;
 * src/marqo/core/constants.py:22-27) as (column, weight) lists, at most 16 each, evaluated in list order in fp64.
 * out_score is the MODIFIED score; order (score desc, doc asc).  B200_ERR_UNSUPPORTED when some document's
 * multiplier is negative on an index with explicit document ids (best chunk != best modified chunk). */
int b200_index_search_modified(b200_index* ix, const float* q, int nq, int k, const int32_t* mult_cols,
                               const double* mult_w, int n_mult, const int32_t* add_cols, const double* add_w, int n_add,
                               int32_t* out_doc, int32_t* out_row, double* out_score);

/* use_external != 0: run this handle's work on the caller's CUDA stream (a cudaStream_t, e.g. torch's current
 * stream; the value 0 is the legacy default stream).  use_external == 0 restores the handle's private stream. */
int b200_index_set_stream(b200_index* ix, void* cuda_stream, int use_external);
/* Device time (ms, CUDA events on the handle's stream) of the scan / merge kernels of the last
 * search call; used by bench.py for the roofline numerator. */
int b200_index_last_timing(b200_index* ix, float* scan_ms, float* merge_ms);
/* Row-sharded corpora: every document number returned by this index is offset by `offset` (the global number of
 * the shard's document 0), so per-shard results can be all-gathered and merged without a fix-up pass. */
int b200_index_set_doc_offset(b200_index* ix, int32_t offset);
/* Device-side merge of all-gathered per-shard results.  d_gathered holds, per shard, the packed block
 * {int32 doc[nq,k] | int32 row[nq,k] | double score[nq,k]} (what b200_index_search_device writes when its three
 * outputs point into one 16*nq*k-byte buffer); blocks are nq*k*16 bytes apart.  nshards*k <= 256. */
int b200_topk_merge_device(b200_index* ix, const void* d_gathered, int nshards, int nq, int k, int32_t* d_out_doc,
                           int32_t* d_out_row, double* d_out_score, int sync);
/* Fused exchange + merge over NVLink peer memory (SURVEY §8e "peer-stores into a symmetric buffer in the top-k
 * epilogue"): one process per GPU; every rank creates an exchange buffer, the ranks swap the 64-byte handles through
 * whatever transport they have (torch.distributed all_gather of a byte tensor), open each other's buffers, and then
 * b200_index_search_exchange = local search + ONE kernel that stores the packed [nq, k] block into every peer's
 * buffer, publishes it with a release flag, waits for the peers' blocks and merges them — no NCCL call on the query
 * path.  All ranks must call it the same number of times with the same nq and k (nq <= 64, world * k <= 256). */
typedef struct b200_exchange b200_exchange;
#define B200_EXCHANGE_HANDLE_BYTES 64
int b200_exchange_create(int device, int rank, int world, int max_nq, int max_k, b200_exchange** out,
                         void* out_handle /* B200_EXCHANGE_HANDLE_BYTES */);
/* handles: world * B200_EXCHANGE_HANDLE_BYTES bytes, rank order (this rank's own entry is ignored). */
int b200_exchange_open(b200_exchange* ex, const void* handles);
int b200_exchange_destroy(b200_exchange* ex);
/* d_local_block: device scratch of nq * k * 16 bytes (this rank's packed block); outputs [nq, k] on the device. */
int b200_index_search_exchange(b200_index* ix, b200_exchange* ex, const float* d_q, int nq, int k, void* d_local_block,
                               int32_t* d_out_doc, int32_t* d_out_row, double* d_out_score, int sync);
/* Merge `nshards` per-shard result lists ([nshards, nq, k] each, host) into the global top-k
 * with the same total order; doc ids must already be global.  Used after the NCCL all-gather
 * of per-shard lists. */
int b200_topk_merge(int nshards, int nq, int k, const int32_t* doc, const int32_t* row, const double* score,
                    int32_t* out_doc, int32_t* out_row, double* out_score);
/* Binary snapshot of the row store (persistence / restart). */
int b200_index_save(b200_index* ix, const char* path);
int b200_index_load(int device, const char* path, b200_index** out);

/* ===================================================================================== */
/* Encoders (SURVEY §8 a2-a5): CLIP ViT image tower, CLIP text tower, BERT (e5).          */
/* Replace model.encode_image / encode_text / AutoModel forward called at                 */
/* src/marqo/core/inference/embedding_models/open_clip_model.py:249-286 and               */
/* src/marqo/core/inference/embedding_models/hugging_face_model.py:172-214.               */
/* ===================================================================================== */

typedef struct b200_model b200_model;

enum b200_arch {
    B200_ARCH_CLIP = 0, /* open_clip CLIP: vision tower + text tower */
    B200_ARCH_BERT = 1, /* HF BertModel + pooling */
    B200_ARCH_MPNET = 2, /* HF MPNetModel + pooling: BERT layers with a relative-position bias in the attention logits */
    B200_ARCH_SIGLIP = 3, /* open_clip SigLIP: class-token-free ViT with a MAP pooling head + bidirectional text tower */
    B200_ARCH_XLMR = 4,   /* HF XLMRobertaModel + pooling: BERT layers, RoBERTa position ids, one token-type row */
    B200_ARCH_CLIP_RESNET = 5, /* OpenAI ResNet CLIP (open_clip ModifiedResNet image tower + the CLIP text tower) */
    B200_ARCH_CLIP_CONVNEXT = 6, /* ConvNeXt CLIP (open_clip TimmModel over a timm ConvNeXt trunk + the CLIP text tower) */
    B200_ARCH_CLIP_EVA = 7, /* EVA02 CLIP (open_clip TimmModel over a timm Eva trunk + the CLIP text tower) */
    B200_ARCH_GTE = 8 /* Alibaba's NewModel (gte-v1.5 architecture, the Stella embedders) + pooling: post-LN layers with
                         rotary q and k and a GeGLU MLP */
};
enum b200_act { B200_ACT_GELU = 0, B200_ACT_QUICKGELU = 1 };
enum b200_pool { B200_POOL_MEAN = 0, B200_POOL_CLS = 1 };

typedef struct b200_tower_desc {
    int32_t width;      /* hidden size: a multiple of 128, <= 1664 for the CLIP towers, <= 1024 for the others */
    int32_t layers;     /* transformer blocks */
    int32_t heads;      /* head_dim = width / heads must be 32 or 64; a CLIP vision tower of at least 128 tokens
                           may also have 80, 88 or 104 (ViT-H-14, ViT-g-14, ViT-bigG-14), which run zero-padded to
                           96, 96 and 128 */
    int32_t mlp;        /* MLP hidden size */
    int32_t ctx;        /* text: context length (77 / 512); vision: unused */
    int32_t vocab;      /* text: vocabulary size; vision: unused */
    int32_t image_size; /* vision: 224 */
    int32_t patch;      /* vision: 32 / 14 */
} b200_tower_desc;

typedef struct b200_model_desc {
    int32_t arch;      /* enum b200_arch */
    int32_t embed_dim; /* output dimension (CLIP projection dim; BERT: == width) */
    int32_t act;       /* enum b200_act */
    int32_t pool;      /* BERT only: enum b200_pool (hugging_face_model.py:205-214) */
    int32_t type_vocab; /* BERT only: token_type vocabulary (2) */
    int32_t max_batch; /* workspace sizing: largest number of items per encode call */
    float image_mean[3]; /* Normalize() constants, src/marqo/s2_inference/clip_utils.py:32-33 */
    float image_std[3];
    b200_tower_desc vision; /* CLIP only */
    b200_tower_desc text;   /* CLIP text tower, or the BERT / MPNet / XLM-R encoder (MPNet, XLM-R: ctx = longest
                               sequence, which is max_position_embeddings - pad_id - 1 because positions start after
                               the pad id) */
    /* MPNet (MPNetConfig), XLM-R and SigLIP: */
    float layer_norm_eps;     /* 1e-5 for the sentence-transformers MPNet checkpoints and XLM-R, 1e-6 for SigLIP */
    /* MPNet and XLM-R: */
    int32_t pad_id;           /* pad_token_id (1): the position ids count from it */
    /* MPNet only: */
    int32_t rel_buckets;      /* relative_attention_num_buckets (32) */
    int32_t rel_max_distance; /* max_distance of relative_position_bucket (128) */
    /* CLIP ResNet only (open_clip ModifiedResNet, verify): the image tower; `vision` is unused.
     *   stem: conv1 3x3 stride 2 (3 -> width/2), conv2 3x3 (width/2 -> width/2), conv3 3x3 (width/2 -> width), each
     *         without bias and followed by BatchNorm (eps 1e-5) and ReLU, then AvgPool2d(2);
     *   stage s = 0..3 of resnet_layers[s] Bottlenecks with planes = width << s, stride 1, 2, 2, 2 on the first block:
     *         ReLU(BN(conv3 1x1 (AvgPool(stride) (ReLU(BN(conv2 3x3 (ReLU(BN(conv1 1x1 (x))))))))) + identity), the
     *         identity being BN(downsample 1x1 conv (AvgPool(stride) (x))) when stride > 1 or the channels change;
     *   attention pool over the (S/32)^2 + 1 tokens [mean; pixels] + positional_embedding, resnet_heads heads of 64,
     *         token 0 out of c_proj, embed_dim wide. */
    int32_t resnet_layers[4];   /* Bottlenecks per stage: RN50 {3, 4, 6, 3}, RN101 {3, 4, 23, 3} */
    int32_t resnet_width;       /* 64 (a power of two >= 64) */
    int32_t resnet_heads;       /* attention-pool heads: width * 32 / 64 (head_dim 64) */
    int32_t resnet_image_size;  /* 224 (a multiple of 32) */
    /* CLIP ConvNeXt only (open_clip TimmModel over timm's ConvNeXt, verify): the image tower; `vision` is unused.
     * Every LayerNorm is over the channels of one pixel, with eps layer_norm_eps (1e-6; 1e-5 for convnext_xxlarge).
     *   stem: Conv2d(3, dims[0], 4, stride 4, bias), LayerNorm;
     *   stage s = 0..3: for s > 0 LayerNorm, Conv2d(dims[s-1], dims[s], 2, stride 2, bias); then depths[s] blocks
     *         x += gamma * fc2(GELU(fc1(LayerNorm(dwconv(x))))), dwconv the 7 x 7 depthwise conv (padding 3, bias),
     *         fc1 dims[s] -> 4 dims[s] and fc2 back, both with bias, GELU the erf one;
     *   head: mean over the pixels, LayerNorm, then convnext_head 0: a Linear without bias to embed_dim, or 1: an MLP
     *         (fc1 with bias to 2 embed_dim, GELU, fc2 without bias to embed_dim).
     * Shapes the kernels cover: dims multiples of 64 up to 3072, convnext_image_size a multiple of 32 up to 640, and
     * embed_dim a multiple of 32; b200_model_create refuses others with B200_ERR_INVALID_ARG. */
    int32_t convnext_dims[4];     /* channels per stage: base {128, 256, 512, 1024}, large {192, ...}, xxlarge {384, ...} */
    int32_t convnext_depths[4];   /* blocks per stage: {3, 3, 27, 3}, xxlarge {3, 4, 30, 3} */
    int32_t convnext_image_size;  /* 224, 256 or 320 */
    int32_t convnext_head;        /* 0: linear projection, 1: MLP */
    /* CLIP ViT: how a uint8 image of another size becomes image_size x image_size: 0 resizes the shortest side and
     * centre-crops (open_clip's default), 1 squashes it, x and y scaled independently without a crop (open_clip's
     * resize_mode "squash": the DFN5B models).  SigLIP always squashes. */
    int32_t resize_squash;
    /* EVA02 CLIP only (open_clip CustomTextCLIP over TimmModel and timm's Eva, verify).  `vision` is the trunk:
     * width <= 1024, head_dim 64, mlp the SwiGLU hidden size H (<= 3072 rounded up to 64: 2048 for EVA02-B-16, 2730
     * for EVA02-L-14), patch, image_size; `text` is the causal CLIP text tower, whose LayerNorms keep eps 1e-5.  Every
     * trunk LayerNorm has eps layer_norm_eps (1e-6).  G = image_size / patch, N = G^2 + 1 tokens:
     *   x = [cls_token; patch_embed(img) + its bias] + pos_embed (no ln_pre);
     *   per block: h = norm1(x); q = h Wq^T + bq, k = h Wk^T (no bias), v = h Wv^T + bv; q and k of tokens 1..N-1 rotated
     *         by the 2-D RoPE below (token 0 is not); o = softmax(q k^T / 8) v per head;
     *         x += attn.proj(attn.norm(o)), attn.norm a LayerNorm over the full width of o;
     *         h = norm2(x); u = SiLU(h Wg^T + bg) * (h Wx^T + bx); x += mlp.fc2(mlp.norm(u)), mlp.norm over the H
     *         columns of u;
     *   head: norm(x) of token 0, head Linear [embed_dim, width] with bias, then the CLIP L2 rule.
     * RoPE (timm RotaryEmbeddingCat, in_pixels False, ref_feat_shape (ref, ref)): the patch at grid row r and column c
     * is token 1 + r G + c, s = ref / G.  In each head, pair i = 0..31 (columns 2i, 2i+1) turns by theta = p 10000^(-j/16)
     * with j = i mod 16, p = r s for i < 16 and c s for i >= 16: (a, b) -> (a cos - b sin, b cos + a sin).  The
     * table is built by the engine (it is not in the checkpoint). */
    int32_t eva_rope_ref_grid;    /* ref_feat_shape: 16 */
    /* GTE only (NewModel with position_embedding_type "rope", verify).  `text` is the encoder: width <= 1024, head_dim
     * 64, mlp the GeGLU hidden size M, ctx <= 512; embed_dim == width; every LayerNorm has eps layer_norm_eps (1e-12);
     * pool as BERT's; token_type_embeddings row 0 is added (type_vocab rows).  Over right-padded ids [B, S]:
     *   x = LN_emb(word[ids] + token_type[0])                        (no position table);
     *   per layer (post-LN): q | k | v = x Wqkv^T + bqkv, heads of 64; q and k of position s = 0..S-1 rotated by the
     *         RoPE below; o = softmax(q k^T / 8 + key mask) v; x = attn_ln(x + o Wo^T + bo);
     *         up | gate = x Wug^T (no bias, up first); x = mlp_ln(x + (GELU_erf(gate) * up) Wd^T + bd);
     *   out = masked mean of x, then F.normalize (as BERT).
     * RoPE (NTKScalingRotaryEmbedding, rotate-half): in each head, pair j = 0..31 (columns j and j + 32) turns by s f_j,
     * f_j = (rope_theta rope_ntk_factor)^(-2j/64) / rope_ntk_factor^(2/64): (a, b) -> (a cos - b sin, b cos + a sin).
     * The table is built by the engine. */
    float rope_theta;             /* 160000 */
    float rope_ntk_factor;        /* rope_scaling factor (type "ntk"): 2; 1 for no scaling */
    /* CoCa (open_clip CoCa, verify), arch B200_ARCH_CLIP.  attn_pool_heads > 0 replaces the vision tower's class-token
     * head with CoCa's attentional pooler over d = embed_dim columns; text_embed_cls != 0 appends CoCa's CLS row to the
     * text.  Every LayerNorm has eps 1e-5.  The image tower, G = image_size / patch, N = G^2 + 1 tokens:
     *   x = the CLIP ViT trunk (conv1 without bias, class token, positional_embedding, ln_pre, the blocks) [N, width];
     *   kv = ln_k(x) over all N rows; q0 = ln_q(query[0]) Wq^T + bq (computed once by b200_model_finalize);
     *   o = MHA(q0, kv Wk^T + bk, kv Wv^T + bv) with attn_pool_heads heads of d / attn_pool_heads (64 or 96) columns,
     *       Wk, Wv [d, width], then out_proj (d -> d, bias);
     *   out = ln_post(o) @ visual.proj [d, embed_dim].
     * Only query 0 is computed (the queries do not interact and the embedding pools query 0).  The text tower over ids
     * [n, ctx - 1] (zero padded): x = [token_embedding[ids] ; cls_emb] + positional_embedding[0..ctx-1], the causal
     * CLIP blocks except that the last row (CLS) keeps key 0 and each key k in 1..ctx-1 with ids[k - 1] != 0; out =
     * ln_final(x[ctx - 1]) @ text_projection.  Both towers then F.normalize (eps 1e-12) every row, always, and divide it
     * by its norm again when normalize is set.  A CLS text tower needs head_dim 64 and ctx <= 127. */
    int32_t attn_pool_heads;      /* 8; 0: the class-token head */
    int32_t text_embed_cls;       /* 1: CoCa's appended CLS row */
    /* M-CLIP's text tower (pt_multilingual_clip MultilingualCLIP, verify), arch B200_ARCH_BERT or B200_ARCH_XLMR with
     * pool B200_POOL_MEAN.  text_proj_dim > 0 replaces the pooling head: the masked mean of the last hidden state over
     * each row's tokens, then LinearTransformation (nn.Linear [text_proj_dim, width] with bias), then, when normalize is
     * set, the division by the L2 norm without an epsilon (the reference's CLIP.normalize).  embed_dim must equal
     * text_proj_dim.  Weights: the encoder's names under an optional "transformer." prefix (dropped), and
     * LinearTransformation.weight [E, width] and LinearTransformation.bias [E].  0: the usual head. */
    int32_t text_proj_dim;
    /* A BERT cross-encoder (transformers BertForSequenceClassification, eval mode; verify), arch B200_ARCH_BERT only.
     * cls_labels > 0 replaces the pooling head: over a pair batch of ids, mask and token-type ids [n, S]
     *   x = LN_emb(word[ids] + token_type[type_ids] + position[s])   (type ids clamped to [0, type_vocab - 1]);
     *   the BERT layers (key mask from attn_mask, erf-GELU);
     *   p = tanh(pooler.dense(x[CLS])), x[CLS] the row of position 0;
     *   out[b] = classifier(p) [cls_labels], then the activation b200_model_classify_tokens asks for.
     * embed_dim must equal cls_labels.  Weights: BertForSequenceClassification's names with the "bert." prefix dropped
     * (embeddings.*, encoder.layer.*, pooler.dense.{weight [W, W], bias}), classifier.{weight [cls_labels, W], bias};
     * b200_model_finalize refuses a missing one with B200_ERR_MISSING_WEIGHT, as every other required parameter.
     * Such a model is run by b200_model_classify_tokens only; b200_model_encode_tokens refuses it with
     * B200_ERR_INVALID_ARG, and b200_model_create refuses cls_labels on any other arch the same way.  0: the usual
     * head. */
    int32_t cls_labels;
    /* OWL-ViT's open-vocabulary detector (transformers OwlViTForObjectDetection, eval mode; verify), arch
     * B200_ARCH_CLIP only, with a CLIP ViT vision tower and the CLIP text tower.  owl_detect = 1 replaces the image
     * embedding head: with G = image_size / patch and the trunk's N = G^2 + 1 token rows x of an image,
     *   e = ln_post(x) (every row);  f_p = layer_norm(e_p * e_0) for the patches p = 1 .. G^2 (row-major, token
     *   1 + r G + c);
     *   logit_p = (c^ . q^ + logit_shift(f_p)) * (ELU(logit_scale(f_p)) + 1), c^ = c / (|c| + 1e-6) for
     *   c = class_head.dense0(f_p) [embed_dim], and q^ = u / (|u| + 1e-6) for the query's unit text embedding
     *   u = t / |t| (t: ln_final of the query's EOT row, at argmax(id), times text_projection);
     *   box_p = sigmoid(box_head.dense2(GELU(dense1(GELU(dense0(f_p))))) + box_bias[p]) as (cx, cy, w, h), box_bias
     *   being the logits of the patch's corner ((c + 1) / G, (r + 1) / G) and of its size 1 / G, each + 1e-4.
     * Weights: the CLIP names of both towers without visual.proj, and the detector's own layer_norm.{weight, bias}
     * [width], class_head.dense0.{weight [embed_dim, width], bias}, class_head.logit_shift.{weight [1, width], bias
     * [1]}, class_head.logit_scale.{weight, bias} (the same shapes), box_head.dense0 / dense1.{weight [width, width],
     * bias} and box_head.dense2.{weight [4, width], bias [4]}; b200_model_finalize refuses a missing one with
     * B200_ERR_MISSING_WEIGHT.  resize_squash must be 1, vision.width <= 1024 and embed_dim + 2 rounded up to 64 at
     * most vision.width.  Such a model is run by b200_model_detect_images_u8 only; every encode call refuses it
     * with B200_ERR_INVALID_ARG.  0: the usual heads. */
    int32_t owl_detect;
    /* LanguageBind's video model (languagebind LanguageBindVideo, eval mode; verify), arch B200_ARCH_CLIP only, with a
     * CLIP ViT of heads of 64 (width <= 1024) and the CLIP text tower.  video_frames = T in 1..16 makes the vision
     * tower a video tower over T frames of N = (image_size / patch)^2 + 1 token rows each, laid out (b T + t) N + token:
     *   x = the CLIP ViT embedding of every frame (conv1 without bias; frame t's class row is class_embedding[t] when
     *       that is [T, width], else class_embedding [width]) + positional_embedding, then ln_pre;
     *   per block, before the CLIP block: x += temporal_embedding[t] on every row of frame t (not when T = 1);
     *       x += out_proj(MHA over the T frames of each (video, token) pair of temporal_ln_1(x)), no mask, heads of 64
     *       with q / k / v / out biases;
     *   head: ln_post of the T class rows, their mean, visual.proj [width, embed_dim], v / |v| * exp(logit_scale), and,
     *       when normalize is set, the division by the norm again (no epsilons).
     * The text tower is the causal CLIP one; its head is LanguageBind's: ln_final of the EOT row (first arg-max id),
     * text_projection, v / |v|, then the division again when normalize is set.  Weights: the CLIP names, visual.proj
     * [width, E], per block visual.transformer.resblocks.{i}.temporal_embedding [T, width], .temporal_ln_1.{weight,
     * bias}, .temporal_attn.in_proj_{weight [3 width, width], bias}, .temporal_attn.out_proj.{weight, bias}, and
     * logit_scale [1].  Such a model encodes uint8 videos by b200_model_encode_videos_u8 and text by the token calls;
     * the image encode calls refuse it with B200_ERR_INVALID_ARG.  0: no video tower. */
    int32_t video_frames;
} b200_model_desc;

int b200_model_create(int device, const b200_model_desc* desc, b200_model** out);
int b200_model_destroy(b200_model* m);
/* Upload one parameter (fp32, host, contiguous) under its checkpoint name: open_clip
 * state_dict names for CLIP ("visual.conv1.weight", "transformer.resblocks.0.attn.in_proj_weight",
 * ...), HF BertModel names for BERT ("embeddings.word_embeddings.weight", ...).  SigLIP: open_clip's names for its
 * timm trunk and text tower (verify): visual.trunk.patch_embed.proj.{weight,bias}, visual.trunk.pos_embed [1, G*G, W],
 * visual.trunk.blocks.{i}.{norm1,attn.qkv,attn.proj,norm2,mlp.fc1,mlp.fc2}.{weight,bias}, visual.trunk.norm.*,
 * visual.trunk.attn_pool.{latent [1, 1, W], q, kv, proj, norm, mlp.fc1, mlp.fc2}.*, text.token_embedding.weight,
 * text.positional_embedding, text.transformer.resblocks.{i}.* (the CLIP block names), text.ln_final.*,
 * text.text_projection.{weight [E, W], bias}. */
/* CoCa: the CLIP ViT names for the trunk (visual.conv1.weight, ..., visual.transformer.resblocks.*), then
 * visual.attn_pool.{query [Q, d] (only row 0 is read; Q = 256 queries), ln_q.* [d], ln_k.* [width],
 * attn.q_proj_weight [d, d], attn.k_proj_weight [d, width], attn.v_proj_weight [d, width], attn.in_proj_bias [3d],
 * attn.out_proj.{weight [d, d], bias}}, visual.ln_post.* [d], visual.proj [d, embed_dim]; the text tower under "text.":
 * text.token_embedding.weight, text.positional_embedding [ctx, W], text.cls_emb [W], text.transformer.resblocks.*,
 * text.ln_final.*, text.text_projection [W, embed_dim].  text.text_decoder.* and logit_scale are not needed. */
/* CLIP ResNet: open_clip ModifiedResNet names (verify): visual.{conv1,conv2,conv3}.weight,
 * visual.{bn1,bn2,bn3}.{weight,bias,running_mean,running_var}, per block visual.layer{1-4}.{i}.{conv1,conv2,conv3}.weight
 * and .bn{1,2,3}.*, the first block's .downsample.0.weight (1x1 conv) and .downsample.1.* (its BatchNorm),
 * visual.attnpool.positional_embedding [(S/32)^2 + 1, 32 width], visual.attnpool.{q,k,v,c}_proj.{weight,bias}; the text
 * tower under the CLIP names.  BatchNorm is folded into the convolutions by b200_model_finalize (num_batches_tracked is
 * not needed). */
/* CLIP ConvNeXt: open_clip TimmModel names (verify): visual.trunk.stem.0.{weight [C0, 3, 4, 4], bias} (the conv),
 * visual.trunk.stem.1.{weight,bias} (its LayerNorm), for s > 0 visual.trunk.stages.{s}.downsample.0.{weight,bias} (the
 * LayerNorm) and .downsample.1.{weight [Cs, Cs-1, 2, 2], bias}, per block visual.trunk.stages.{s}.blocks.{i}.conv_dw.{weight
 * [C, 1, 7, 7], bias}, .norm.*, .mlp.fc1.*, .mlp.fc2.* and .gamma [C], visual.trunk.head.norm.{weight,bias}, then
 * visual.head.proj.weight [E, C3] (linear head) or visual.head.mlp.{fc1.weight [2E, C3], fc1.bias, fc2.weight [E, 2E]}
 * (MLP head); the text tower under the CLIP names.  b200_model_finalize folds gamma into fc2's rows and bias. */
/* XLM-R: HF XLMRobertaModel names, as BERT's: embeddings.word_embeddings.weight [vocab, W],
 * embeddings.position_embeddings.weight [ctx + pad_id + 1, W], embeddings.token_type_embeddings.weight [1, W],
 * embeddings.LayerNorm.*, encoder.layer.{i}.* (a "roberta." prefix is dropped). */
/* GTE: NewModel names (verify): embeddings.word_embeddings.weight [vocab, W], embeddings.token_type_embeddings.weight
 * [type_vocab, W], embeddings.LayerNorm.*, per layer encoder.layer.{i}.attention.qkv_proj.{weight [3W, W], bias},
 * .attention.o_proj.{weight,bias}, .attn_ln.{weight,bias}, .mlp.up_gate_proj.weight [2M, W] (up rows, then gate rows;
 * no bias), .mlp.down_proj.{weight [W, M], bias}, .mlp_ln.{weight,bias} (a "new." prefix is dropped; pooler weights are
 * not needed).  An up_gate_proj without 2 text.mlp rows is refused with B200_ERR_INVALID_ARG. */
/* CLIP EVA02: open_clip CustomTextCLIP names over TimmModel (verify): visual.trunk.patch_embed.proj.{weight [W, 3, P, P],
 * bias}, visual.trunk.cls_token [1, 1, W], visual.trunk.pos_embed [1, N, W], per block visual.trunk.blocks.{i}.norm1.*,
 * .attn.q_proj.{weight,bias}, .attn.k_proj.weight, .attn.v_proj.{weight,bias}, .attn.norm.*, .attn.proj.*, .norm2.*,
 * .mlp.fc1_g.{weight [H, W], bias}, .mlp.fc1_x.*, .mlp.norm.{weight,bias} [H], .mlp.fc2.{weight [W, H], bias},
 * visual.trunk.norm.*, visual.trunk.head.{weight [E, W], bias}; the text tower under the CLIP block names with a
 * "text." prefix (text.token_embedding.weight, ..., text.ln_final.*) and text.text_projection [W, E].
 * b200_model_finalize fuses q | k | v (k with a zero bias), folds the patch bias into pos_embed's patch rows, fuses
 * fc1_g | fc1_x with the hidden size padded to a multiple of 64 by zero rows (and fc2 by zero columns), and builds the
 * RoPE table.  A checkpoint whose fc1_g has other than vision.mlp rows is refused with B200_ERR_INVALID_ARG. */
int b200_model_load_tensor(b200_model* m, const char* name, const float* data, int64_t numel);
/* Verifies every required parameter has been supplied, builds derived buffers. */
int b200_model_finalize(b200_model* m);

/* Images as uint8 HWC (host), all n of size h x w: resize (bicubic, shortest side) ->
 * centre-crop -> /255 -> Normalize -> ViT -> proj -> optional L2 normalise.
 * Replaces preprocessors['image'](pil).to(device) (src/marqo/tensor_search/add_docs.py:129-134)
 * + OPEN_CLIP.encode_image (open_clip_model.py:249-266).  out: fp32 host [n, embed_dim].
 * The /255 and Normalize steps happen inside the patch-embedding GEMM's operand load (its gather warps read the uint8
 * pixels and write bf16 into the tensor core's shared-memory operand): no normalised image or patch matrix exists in HBM
 * (SURVEY §8 a2; images already of the model's size skip the resize pass as well). */
int b200_model_encode_images_u8(b200_model* m, const uint8_t* hwc, int n, int h, int w, int normalize,
                                float* out);
/* Already-preprocessed fp32 CHW tensors [n,3,S,S] (the reference passes these through
 * unchanged: abstract_clip_model.py:108-111). */
int b200_model_encode_images_f32(b200_model* m, const float* chw, int n, int normalize, float* out);
/* SigLIP images: the resize squashes the image to S x S (independent x and y scales, no crop); the tower has no class
 * token and pools with its MAP head (embed_dim == vision width, no projection). */
/* Token ids int32 [n, seq] (host).  CLIP: causal text tower, EOT = arg-max id pooling.  CoCa (text_embed_cls): seq
 * must be text.ctx - 1 (76), the CLS row is appended and pooled; attn_mask is ignored.
 * SigLIP: bidirectional text tower (no mask), the last position of each row is pooled, then ln_final and the biased
 * text projection; attn_mask is ignored (the tokenizer pads every row to the context length).
 * BERT: attn_mask int32 [n, seq] (1 = token, 0 = pad; NULL = all ones), token_type 0.
 * MPNet: as BERT, without token types; position ids follow the ids (HF create_position_ids_from_input_ids), the key
 * mask follows attn_mask.  XLM-R: as MPNet, plus token_type_embeddings row 0, LayerNorm eps layer_norm_eps.
 * GTE: as BERT, without a position table; q and k rotated by position.
 * seq > text.ctx is refused with B200_ERR_INVALID_ARG. */
int b200_model_encode_tokens(b200_model* m, const int32_t* ids, const int32_t* attn_mask, int n, int seq,
                             int normalize, float* out);
/* Device-resident variants: inputs/outputs are device pointers on the model's device,
 * asynchronous on the model's stream unless sync != 0. */
int b200_model_encode_images_u8_device(b200_model* m, const uint8_t* d_hwc, int n, int h, int w, int normalize,
                                       float* d_out, int sync);
int b200_model_encode_tokens_device(b200_model* m, const int32_t* d_ids, const int32_t* d_attn_mask, int n,
                                    int seq, int normalize, float* d_out, int sync);
/* A cross-encoder's scores (cls_labels > 0, see b200_model_desc): sentence pairs as ids, attn_mask (NULL: all ones, else
 * a right-padded prefix mask as b200_model_encode_tokens takes) and type_ids (0 up to the first [SEP], 1 after it;
 * NULL: all 0), each int32 [n, seq] on the host.  activation 0 returns the logits, 1 their sigmoid
 * (sentence-transformers' CrossEncoder default for one label).  out: fp32 host [n, cls_labels].  A model without a
 * classification head, or any other activation: B200_ERR_INVALID_ARG. */
int b200_model_classify_tokens(b200_model* m, const int32_t* ids, const int32_t* attn_mask, const int32_t* type_ids,
                               int n, int seq, int activation, float* out);
/* The same with device-resident inputs and output, asynchronous on the model's stream unless sync != 0. */
int b200_model_classify_tokens_device(b200_model* m, const int32_t* d_ids, const int32_t* d_attn_mask,
                                      const int32_t* d_type_ids, int n, int seq, int activation, float* d_out, int sync);
/* OWL-ViT detection (owl_detect = 1, see b200_model_desc): one text query, query_ids int32 [seq] on the host (seq <=
 * text.ctx), scored against each of n uint8 HWC images [h, w, 3] (hwc, host), which are squashed to image_size by the
 * Pillow-exact resize.  logits: fp32 host [n, G^2], what OwlViTForObjectDetection returns as logits[..., 0]; boxes: fp32
 * host [n, G^2, 4], its pred_boxes (cx, cy, w, h in [0, 1]).  n larger than the batch the workspaces hold runs in
 * sub-batches.  A model without the detector, seq outside 1 .. text.ctx, or n, h or w <= 0: B200_ERR_INVALID_ARG. */
int b200_model_detect_images_u8(b200_model* m, const uint8_t* hwc, int n, int h, int w, const int32_t* query_ids,
                                int seq, float* logits, float* boxes);
/* LanguageBind videos (video_frames > 0, see b200_model_desc): n videos of t frames, uint8 RGB thwc [n, t, h, w, 3]
 * (host), t == video_frames.  Each frame goes through LanguageBind's video transform on the GPU (ShortSideScale to
 * image_size, bilinear, align_corners False, no antialias; CenterCropVideo with Python's round; / 255; Normalize by
 * image_mean / image_std; the training-time random horizontal flip the reference also applies is not), then the video
 * tower.  out: fp32 host [n, embed_dim].  A model without a video tower, t != video_frames, or n, h or w <= 0:
 * B200_ERR_INVALID_ARG. */
int b200_model_encode_videos_u8(b200_model* m, const uint8_t* thwc, int n, int t, int h, int w, int normalize,
                                float* out);
/* The same with the videos and the output on the model's device, asynchronous on its stream unless sync != 0. */
int b200_model_encode_videos_u8_device(b200_model* m, const uint8_t* d_thwc, int n, int t, int h, int w, int normalize,
                                       float* d_out, int sync);
/* Images of mixed sizes in one call (every vision tower that takes uint8 images): image i is uint8 HWC
 * [heights[i], widths[i], 3] at hwc[i]; hwc, heights and widths are host arrays of n.  The images are resized to the
 * model's S x S by the tower's rule (shortest side + centre crop, or the squash) in one pass over each sub-batch, two
 * kernels whatever the mix of sizes, and the tower runs once per sub-batch; images already S x S pass through
 * unchanged.  out: fp32 host [n, embed_dim], row i for image i.  The host variant copies each sub-batch's images to the
 * device, one copy per run of images that lie back to back in host memory.  NULL arrays or entries, n <= 0, a height
 * or width <= 0, or a model without a vision tower: B200_ERR_INVALID_ARG, nothing written. */
int b200_model_encode_images_u8_ragged(b200_model* m, const uint8_t* const* hwc, const int32_t* heights,
                                       const int32_t* widths, int n, int normalize, float* out);
/* The same with device-resident images: d_hwc is a host array of n device pointers on the model's device; d_out fp32
 * device [n, embed_dim]; asynchronous on the model's stream unless sync != 0 (the call's host-side tables have been
 * uploaded by the time it returns). */
int b200_model_encode_images_u8_ragged_device(b200_model* m, const uint8_t* const* d_hwc, const int32_t* heights,
                                              const int32_t* widths, int n, int normalize, float* d_out, int sync);
int b200_model_set_stream(b200_model* m, void* cuda_stream, int use_external);
/* Optional per-kernel-class device timing: when enabled every GEMM / attention launch of an encode call is
 * bracketed by CUDA events on the handle's stream; b200_model_profile returns their sums over every encode call
 * since profiling was last (re-)enabled. */
int b200_model_set_profiling(b200_model* m, int enable);
int b200_model_profile(b200_model* m, float* gemm_ms, int* gemm_launches, float* attention_ms, int* attention_launches);
/* Device time (ms) of the last encode call and the number of kernels it launched. */
int b200_model_last_timing(b200_model* m, float* ms, int* launches);

/* Weighted-mean fusion + renormalise on the host-side contract of
 * src/marqo/tensor_search/tensor_search.py:1953-1973 and
 * src/marqo/core/inference/tensor_fields_container.py:355-365:
 * out = mean_i(w_i * v_i); if normalize and |out| > 0: out /= |out|.  fp64 arithmetic. */
int b200_fuse_vectors(const double* vecs, const double* weights, int n, int dim, int normalize, double* out);

/* ===================================================================================== */
/* Tokenizers (SURVEY §8 f2): text -> int32 token ids on the host, multi-threaded.       */
/* ===================================================================================== */

typedef struct b200_tokenizer b200_tokenizer;

/* WordPiece — what AutoTokenizer.from_pretrained(<BERT / e5 checkpoint>) gives the reference
 * (src/marqo/core/inference/embedding_models/hugging_face_model.py:125-130) and what encode() calls as
 * tokenizer(sentences, padding=True, truncation=True, max_length=...) (:179-185).  vocab_utf8: the bytes of vocab.txt
 * (one token per line, id = line number; must contain [PAD] [UNK] [CLS] [SEP]).  do_lower_case != 0 also strips
 * accents (BertNormalizer's strip_accents=None follows lowercase). */
int b200_tokenizer_create_wordpiece(const char* vocab_utf8, size_t nbytes, int do_lower_case, b200_tokenizer** out);
/* The same WordPiece with the special tokens named by the caller: rows are "cls ids sep", padded with `pad`, words
 * without a piece become `unk`, and exactly the n_specials strings of `specials` are matched verbatim in the raw text
 * (MPNetTokenizer: "<s>", "</s>", "<pad>", "[UNK]" and specials <s> <pad> </s> [UNK] <mask>).  Every named token must be
 * in the vocabulary. */
int b200_tokenizer_create_wordpiece_ex(const char* vocab_utf8, size_t nbytes, int do_lower_case, const char* cls,
                                       const char* sep, const char* pad, const char* unk, const char* const* specials,
                                       int n_specials, b200_tokenizer** out);
/* CLIP byte-level BPE — open_clip's SimpleTokenizer, the tokenizer OPEN_CLIP.load_tokenizer() returns for non-hf-hub
 * models (src/marqo/core/inference/embedding_models/open_clip_model.py:211-222; cleaning rules restated at
 * src/marqo/core/inference/embedding_models/hf_tokenizer.py:9-17).  merges_utf8: the DECOMPRESSED bytes of
 * bpe_simple_vocab_16e6.txt (line 1 is a header; at most 49152-256-2 merges are used).  ftfy.fix_text is not
 * restated: text that ftfy would repair (mojibake) tokenises as written. */
int b200_tokenizer_create_clip_bpe(const char* merges_utf8, size_t nbytes, b200_tokenizer** out);
/* SentencePiece Unigram with XLM-RoBERTa's ids — XLMRobertaTokenizer on sentencepiece.bpe.model.  model_bytes: the
 * serialized ModelProto (model_type UNIGRAM; no user-defined pieces).  Normalisation: the precompiled charsmap (longest
 * match, the character itself when nothing matches), remove_extra_whitespaces, add_dummy_prefix, spaces -> U+2581;
 * segmentation: Viterbi over the pieces, an unknown character scores min_score - 10 and adjacent unknowns merge.
 * Ids: <s> 0, <pad> 1, </s> 2, <unk> 3, any other piece its SentencePiece id + 1 (fairseq's offset); vocab_size is
 * pieces + 2 (<pad> and <mask>).  Special-token strings in the text are ordinary text. */
int b200_tokenizer_create_unigram(const char* model_bytes, size_t nbytes, b200_tokenizer** out);
int b200_tokenizer_destroy(b200_tokenizer* t);
int b200_tokenizer_vocab_size(b200_tokenizer* t, int* out_size);
/* Encode n UTF-8 strings (texts[i], text_bytes[i] bytes; invalid sequences decode as U+FFFD).
 * WordPiece: "[CLS] ids [SEP]" (Unigram: "<s> ids </s>", padded with <pad>), truncated to max_length, every row padded with [PAD] to the LONGEST row of this call
 * (padding=True): *out_seq_len = that length <= max_length.  CLIP BPE: "<start_of_text> ids <end_of_text>", truncated
 * to max_length (= context_length) with the last id forced to <end_of_text>, zero padded: *out_seq_len = max_length.
 * out_ids / out_mask (mask may be NULL): caller buffers of n * max_length int32; rows are written back to back with
 * stride *out_seq_len.  max_length >= 2.  Thread-safe (the handle is immutable after creation). */
int b200_tokenizer_encode(b200_tokenizer* t, const char* const* texts, const int64_t* text_bytes, int n, int max_length,
                          int32_t* out_ids, int32_t* out_mask, int* out_seq_len);
/* WordPiece sentence pairs, what a cross-encoder's tokenizer(texts_a, texts_b, padding=True, truncation='longest_first',
 * max_length=max_length) gives: row i is "[CLS] A [SEP] B [SEP]" for A = texts_a[i], B = texts_b[i], type ids 0 through
 * the first [SEP] and 1 after it, padded with [PAD] (type 0, mask 0) to the longest row of the call.  Truncation is
 * HF tokenizers' longest_first over the budget m = max_length - 3: with n1 <= n2 the two lengths (the shorter first),
 * when n1 + n2 > m, n2 = n1 if n1 > m, else max(n1, m - n1); if n1 + n2 is still over m, n1 = m / 2 and n2 = n1 + m % 2;
 * each side then keeps its first min(its length, its share) ids.  out_ids, out_mask, out_type_ids (mask and type ids
 * may be NULL): caller buffers of n * max_length int32, rows back to back with stride *out_seq_len.  max_length >= 3.
 * WordPiece tokenizers only (B200_ERR_INVALID_ARG otherwise). */
int b200_tokenizer_encode_pairs(b200_tokenizer* t, const char* const* texts_a, const int64_t* bytes_a,
                                const char* const* texts_b, const int64_t* bytes_b, int n, int max_length,
                                int32_t* out_ids, int32_t* out_mask, int32_t* out_type_ids, int* out_seq_len);

/* Recommender interpolation (SURVEY §8 f3): src/marqo/core/utils/vector_interpolation.py —
 * Lerp.interpolate :49-88 (sum_i (w_i / sum w) v_i), Nlerp.interpolate :91-119 (Lerp, then / |.|),
 * Slerp hierarchical :121-193,211-237.  vecs: fp64 [n, dim] host; out: fp64 [dim].  Host-side fp64 arithmetic in
 * the reference's order (these are <= a few dozen vectors per recommend call, src/marqo/core/search/recommender.py:88).
 * On the reference's error conditions returns B200_ERR_INVALID_ARG and stores which one in *out_error_kind so the
 * binding can raise ZeroSumWeightsError / ZeroMagnitudeVectorError / ValueError like the reference. */
enum b200_interp_method { B200_INTERP_LERP = 0, B200_INTERP_NLERP = 1, B200_INTERP_SLERP = 2 };
enum b200_interp_error {
    B200_INTERP_OK = 0,
    B200_INTERP_ZERO_SUM_WEIGHTS = 1, /* ZeroSumWeightsError      (:12, :74-77, :226-228) */
    B200_INTERP_ZERO_MAGNITUDE = 2,   /* ZeroMagnitudeVectorError (:16, :113-116) */
    B200_INTERP_ZERO_LENGTH = 3       /* ValueError               (:171-173) */
};
int b200_interpolate_vectors(const double* vecs, const double* weights, int n, int dim, int method, double* out,
                             int* out_error_kind);

/* ===================================================================================== */
/* Image decode (SURVEY §8 f4): baseline JPEG -> uint8 HWC RGB on the GPU.               */
/* Replaces the Pillow decode on Marqo's download threads (Image.open at                  */
/* src/marqo/core/inference/image_download.py:146-152, pixels materialised by the         */
/* transform at src/marqo/tensor_search/add_docs.py:129-134).  Huffman decoding runs on   */
/* the host (images of a batch in parallel); dequantisation + integer IDCT, fancy chroma  */
/* upsampling and YCbCr -> RGB run in two CUDA kernels over the whole batch and reproduce */
/* libjpeg-turbo's default decode (what Pillow returns) bit for bit.                      */
/* ===================================================================================== */

/* Size of a JPEG and whether this decoder handles it (baseline / extended-sequential Huffman, 8-bit, grey or YCbCr
 * with 4:4:4 / 4:2:2 / 4:2:0 sampling).  *out_supported == 0: decode it with Pillow (b200_last_error says why). */
int b200_jpeg_info(const uint8_t* file, size_t nbytes, int32_t* out_height, int32_t* out_width, int32_t* out_supported);
/* Decode n files.  d_out[i]: device buffer of heights[i] * widths[i] * 3 bytes on `device` (sizes from b200_jpeg_info, or
 * from a first call with d_out[i] == NULL, which only fills heights / widths / status).  status[i]: B200_OK,
 * B200_ERR_UNSUPPORTED (fall back to Pillow for this image) or B200_ERR_INVALID_ARG (no output buffer).  Synchronous. */
int b200_jpeg_decode_batch(int device, const uint8_t* const* files, const size_t* nbytes, int n, uint8_t* const* d_out,
                           int32_t* heights, int32_t* widths, int32_t* status);

/* ===================================================================================== */
/* Diagnostics: run ONE kernel of the encoder (used by the kernel-level numerics tests;  */
/* not part of the reference-facing surface).  The hooks with a `stream` argument take   */
/* device buffers on `device`, bf16 ones typed void*, except where a comment says host;  */
/* they run on `stream` (a cudaStream_t, 0: the legacy default stream) and synchronise   */
/* it before they return.                                                                */
/* ===================================================================================== */

/* out = act(A @ W^T + bias) (+ residual) over rows [0, M) x columns [0, N): A bf16 [M, lda], W bf16 [N, K], fp32
 * accumulate; act: 0 none, 1 erf-GELU, 2 QuickGELU; bias fp32 [N] and residual fp32 [M, ldr] may be NULL, and residual
 * may be out itself (fp32 only), as the encoder layers update their residual stream.  out [M, ldo] is bf16 when
 * out_bf16 != 0, fp32 otherwise.  The library picks the kernel by its usual rule for an SM count of sms (0: the
 * device's own); *kernel_out (when not NULL) receives the kernel it ran: 0 the 128 x 128 tiles, 1 the persistent
 * 128 x 256 tiles. */
int b200_debug_gemm(int device, const void* A, int lda, const void* W, const float* bias, const float* residual, int ldr,
                    void* out, int ldo, int out_bf16, int act, int M, int N, int K, int sms, int* kernel_out,
                    void* stream);
/* Scan kernel of a row store.  force_streamed: 1 makes every later search of ix scan with the streamed-query kernel
 * whatever its dim (so both kernels can run on one corpus), 0 restores the library's rule (resident query block up to
 * dim 1024, streamed above), -1 leaves the setting unchanged.  *last_kernel (when not NULL) receives the kernel the last
 * search ran: 0 resident query block, 1 streamed query block, -1 no search yet. */
int b200_debug_index_scan_kernel(b200_index* ix, int force_streamed, int* last_kernel);
/* What the last search of ix left on the device for its last query group (read only: no search state changes).
 * *nq and *grid (when not NULL) receive the group's size and the scan's grid, both 0 before any scan.  Each array
 * that is not NULL receives, for that group: eps fp32 [nq], the per-query bound on |approximate - exact| scan key;
 * queries fp32 [nq, dim], the fp16 query block as it was scanned; list_score fp32, list_row and list_doc int32
 * [grid, nq, 16], every scan CTA's sorted list of its 16 best (approximate key, row, document) per query, unused
 * entries -inf / -1 / -1.  The collect pass and the merge do not write the lists, so the keys are the scan's. */
int b200_debug_index_last_scan(b200_index* ix, int* nq, int* grid, float* eps, float* queries, float* list_score,
                               int32_t* list_row, int32_t* list_doc);
/* Mean device time (ms, CUDA events) of `iters` back-to-back GEMM launches [M,K] x [N,K]^T on device-generated data,
 * with the epilogue given by act, out_bf16, has_bias and residual_in_place (residual == out, fp32 only). */
int b200_debug_gemm_time(int device, int M, int N, int K, int act, int out_bf16, int has_bias, int residual_in_place,
                         int iters, float* out_ms);
/* The patch embedding of uint8 HWC images [n,S,S,3] (G = (S/patch)^2 patches each) by the fused gather GEMM: each
 * patch is ToTensor + Normalize (mean3/std3, host fp32 [3])-ed inside the operand load, no patch matrix in HBM
 * (src/marqo/tensor_search/add_docs.py:129-134), and conv1 is conv_w fp32 [N, 3*patch*patch] without bias.  The
 * three forms the image forwards run:
 *   pos != NULL, the ViT form (CLIP, EVA02, the big ViTs, SigLIP): the token rows fed to ln_pre, T = G + (cls != NULL)
 *     per image, out fp32 [n*T, N] (ldo == N): with a class row (cls fp32 [N]) row b*T = cls + pos[0] and row
 *     b*T+1+i = conv1(patch i of image b) + pos[1+i]; without one (SigLIP) row b*T+i = conv1(patch i) + pos[i].
 *     pos fp32 [T, N]; bias must be NULL.
 *   pos == NULL, the ConvNeXt stem form: row b*G+i of out fp32 [n*G, ldo] (ldo >= N, a multiple of 8) =
 *     conv1(patch i of image b) + bias (fp32 [N], NULL: none); cls must be NULL.
 * Nothing of out outside those n*T or n*G rows and their first N columns is written. */
int b200_debug_patch_embed(int device, const uint8_t* hwc, int n, int S, int patch, const float* conv_w, int N,
                           const float* mean3, const float* std3, const float* cls, const float* pos,
                           const float* bias, float* out, int ldo, void* stream);
/* softmax(q k^T / sqrt(head_dim) + mask + bias) v over packed qkv bf16 [B*S, 3*W], head_dim = W / H (32 or 64);
 * mask: 0 none, 1 causal, 2 key length (kv_len int32 [B]), 3 CoCa's CLS mask (kv_len: the ids int32 [B, S - 1]; causal,
 * and the last row keeps key 0 and each key k with ids[b, k - 1] != 0; head_dim 64, S < 128).  rel_bias (NULL: none) is MPNet's relative-position bias,
 * a host array fp32 [H, 2*smax - 1] (natural-log domain, as it enters softmax): rel_bias[h, j - i + smax - 1] is added
 * to the logit of query i and key j; head_dim 64, mask 2, S <= smax.  out bf16 [B*S, W]. */
int b200_debug_attention(int device, const void* qkv, int B, int S, int W, int H, int mask, const int32_t* kv_len,
                         const float* rel_bias, int smax, void* out, void* stream);
/* b200_debug_attention (without a bias) over heads of W / H columns whose logits take the scale 1 / sqrt(model_hd):
 * the zero-padded heads of the ViT-H / g / bigG vision towers (model_hd 80, 88 or 104 in heads of 96 or 128). */
int b200_debug_attention_padded(int device, const void* qkv, int B, int S, int W, int H, int model_hd, int mask,
                                const int32_t* kv_len, void* out, void* stream);
/* MPNet's relative_position_bucket as the model builds its bias table: out[d + max_len - 1] = bucket of
 * key - query = d for |d| < max_len (host-only). */
int b200_debug_relative_position_buckets(int num_buckets, int max_distance, int max_len, int32_t* out);
/* Mean device time (ms, CUDA events) of `iters` back-to-back attention launches on device-generated data, every key
 * kept; rel_bias != 0 adds a generated relative-position bias table with smax = S (the bias runs with mask 2). */
int b200_debug_attention_time(int device, int B, int S, int W, int H, int mask, int rel_bias, int iters, float* out_ms);
/* LayerNorm over `rows` rows of width w, row r read at x + r * in_stride (0: w); x holds (rows - 1) * in_stride + w
 * floats.  out_f32 (fp32) and out_bf16 (bf16), either may be NULL but not both, receive the output [rows, w].
 * out_f32 == x normalises in place (needs in_stride == w). */
int b200_debug_layernorm(int device, const float* x, long long in_stride, const float* gamma, const float* beta, float eps,
                         int rows, int w, float* out_f32, void* out_bf16, void* stream);
/* b200_debug_layernorm over bf16 rows x (EVA02's attn.norm): out bf16 [rows, w]; w a multiple of 128, <= 1664. */
int b200_debug_layernorm_bf16(int device, const void* x, long long in_stride, const float* gamma, const float* beta,
                              float eps, int rows, int w, void* out, void* stream);
/* EVA02's rotary embedding in place on qkv bf16 [n*S, 3w] (heads of 64, S = G^2 + 1 tokens per image), with the
 * (cos, sin) table the model builds for grid G and reference grid ref (see b200_model_desc).  Class rows and v
 * columns are left as they are. */
int b200_debug_rope_qk(int device, void* qkv, int n, int G, int w, int ref, void* stream);
/* GTE's rotary embedding in place on qkv bf16 [n*S, 3w] (heads of 64): rotate-half pairs (columns j, j + 32) of every
 * row's q and k, position s = 0..S-1 of each sequence, with the table the model builds from rope_theta = theta and
 * rope_ntk_factor = ntk_factor (see b200_model_desc).  v columns are left as they are. */
int b200_debug_rope_qk_half(int device, void* qkv, int n, int S, int w, float theta, float ntk_factor, void* stream);
/* GTE's GeGLU: in bf16 [rows, 2h] (up | gate) -> out bf16 [rows, h] = GELU_erf(gate) * up at row stride ldo (out may be
 * in with ldo = 2h).  h a multiple of 8. */
int b200_debug_geglu(int device, const void* in, int rows, int h, void* out, long long ldo, void* stream);
/* EVA02's SwiGLU + LayerNorm: in bf16 [rows, 2 hp] (gate | x, hp = h rounded up to 64), gamma / beta fp32 [h] ->
 * out bf16 [rows, hp] at row stride ldo (out may be in with ldo = 2 hp), pad columns 0. */
int b200_debug_swiglu_ln(int device, const void* in, int rows, int h, const float* gamma, const float* beta, float eps,
                         void* out, long long ldo, void* stream);
/* CLIP / SigLIP text embedding: x fp32 [n*S, w] = tok[ids] + pos[s], eot int32 [n] = first arg-max of each ids row.
 * tok [vocab, w], pos [S, w]. */
int b200_debug_clip_text_embed(int device, const int32_t* ids, const float* tok, const float* pos, int n, int S, int w,
                               int vocab, float* x, int32_t* eot, void* stream);
/* CoCa's text embedding: ids int32 [n, S - 1], x fp32 [n*S, w] with row s < S - 1 of sequence b = tok[ids[b, s]] +
 * pos[s] and row S - 1 = cls [w] + pos[S - 1]; eot int32 [n] = S - 1. */
int b200_debug_clip_text_embed_cls(int device, const int32_t* ids, const float* tok, const float* pos, const float* cls,
                                   int n, int S, int w, int vocab, float* x, int32_t* eot, void* stream);
/* Embedding + LayerNorm: x fp32 [n*S, w] = LN(word[ids] + type0 + pos[p]), h bf16 [n*S, w] its bf16 copy, kv_len int32
 * [n] = sum of each mask row (S when mask is NULL).  pad < 0: BERT, p = s, type0 [w] required, pos_rows >= S, or pos
 * NULL for no position row (GTE).
 * pad >= 0: RoBERTa (XLM-R with type0, MPNet with type0 NULL), HF's position ids counted from the ids and pad,
 * pos_rows >= pad + S + 1.
 * type_ids (BERT with positions only; NULL: none): int32 [n, S], and type0 is then the whole token-type table
 * [type_rows, w], row type_ids[b, s] (clamped to [0, type_rows - 1]) added in place of row 0. */
int b200_debug_embed_ln(int device, const int32_t* ids, const int32_t* mask, const float* word, const float* pos,
                        int pos_rows, const float* type0, const float* gamma, const float* beta, float eps, int n, int S,
                        int w, int vocab, int pad, float* x, void* h, int32_t* kv_len, const int32_t* type_ids,
                        int type_rows, void* stream);
/* CLIP head over token rows x fp32 [n*S, w]: LN(row b*S + row_in_seq[b]) @ proj [w, E] (row_in_seq NULL: row 0;
 * every entry must lie in [0, S)), divided by its L2 norm if normalize.  out fp32 [n, E]. */
int b200_debug_clip_head(int device, const float* x, int S, const int32_t* row_in_seq, const float* gamma,
                         const float* beta, float eps, const float* proj, int n, int w, int E, int normalize, float* out,
                         void* stream);
/* BERT head over x fp32 [n*S, w]: mean of the first kv_len[b] rows (pool 0) or row 0 (pool 1), then F.normalize if
 * normalize.  out fp32 [n, w]. */
int b200_debug_bert_head(int device, const float* x, const int32_t* kv_len, int n, int S, int w, int pool, int normalize,
                         float* out, void* stream);
/* M-CLIP's text head over x fp32 [n*S, w]: the mean of the first kv_len[b] rows, then @ proj [w, E] (the transposed
 * LinearTransformation.weight) + bias [E] (NULL: none), divided by its L2 norm if normalize.  out fp32 [n, E].
 * w a multiple of 4, <= 1024. */
int b200_debug_text_head(int device, const float* x, const int32_t* kv_len, int n, int S, int w, const float* proj,
                         const float* bias, int E, int normalize, float* out, void* stream);
/* OWL-ViT's patch features over the trunk rows x fp32 [n*N, w] (N = G^2 + 1 rows per image, class row first):
 * out[b*G^2 + p - 1] = LN_det(LN_post(x[b*N + p]) * LN_post(x[b*N])) for p = 1 .. G^2, LN_post by post_g / post_b and
 * LN_det by det_g / det_b (both eps).  out bf16 [n*G^2, w].  w a multiple of 128, <= 1024. */
int b200_debug_owl_merge_ln(int device, const float* x, int n, int N, int w, const float* post_g, const float* post_b,
                            const float* det_g, const float* det_b, float eps, void* out, void* stream);
/* OWL-ViT's class logits from the class head GEMM's rows c fp32 [M, ldc] (columns 0 .. E-1 dense0 with its bias, E
 * logit_shift, E + 1 logit_scale) and the query's text embedding t fp32 [E] (not normalised): out[r] = (c^ . q^ +
 * shift) * (ELU(scale) + 1) with c^ = c / (|c| + 1e-6), u = t / |t| and q^ = u / (|u| + 1e-6).  out fp32 [M]. */
int b200_debug_owl_class_logits(int device, const float* c, int ldc, int M, int E, const float* t, float* out,
                                void* stream);
/* OWL-ViT's boxes from the box head's second hidden rows a bf16 [M, w] (after its GELU): out[r, j] = sigmoid(w2[j] . a[r]
 * + b2[j] + box_bias[r % P, j]) for w2 fp32 [4, w], b2 [4], box_bias fp32 [P, 4].  out fp32 [M, 4]. */
int b200_debug_owl_boxes(int device, const void* a, int M, int w, int P, const float* w2, const float* b2,
                         const float* box_bias, float* out, void* stream);
/* OWL-ViT's box bias of a G x G grid as the model builds it, in fp64 rounded to fp32 (host-only): out fp32 [G^2, 4],
 * row r G + c = (logit((c + 1) / G), logit((r + 1) / G), logit(1 / G), logit(1 / G)) with logit(v) = log(v + 1e-4) -
 * log1p(-v + 1e-4). */
int b200_debug_owl_box_bias(int G, float* out);
/* BertForSequenceClassification's head over x fp32 [n*S, w]: p = tanh(pool_w [w, w] . x[b*S] + pool_b [w]), then
 * out[b, l] = cls_w[l] . p + cls_b[l] for cls_w [L, w], cls_b [L], through the sigmoid if sigmoid != 0.  out fp32
 * [n, L].  w <= 1024. */
int b200_debug_cls_head(int device, const float* x, int n, int S, int w, const float* pool_w, const float* pool_b,
                        const float* cls_w, const float* cls_b, int L, int sigmoid, float* out, void* stream);
/* LanguageBind's heads over x fp32 [n*T*N, w]: for item b the mean over t < T of LN(x[(b T + t) N + r]) (r =
 * row_in_seq[b], NULL: 0; gamma, beta, eps) @ proj [w, E], then v / |v| * scale, then / its norm if normalize.  The
 * video head is r = 0 with scale exp(logit_scale); the text head T = 1, r = the EOT row, scale 1.  out fp32 [n, E]. */
int b200_debug_frame_mean_head(int device, const float* x, int N, int T, const int32_t* row_in_seq, const float* gamma,
                               const float* beta, float eps, const float* proj, int n, int w, int E, float scale,
                               int normalize, float* out, void* stream);
/* LanguageBind's temporal step over x fp32 [rows, w] (rows (b T + t) N + token): x[r] += temb[(r / N) % T] in place
 * (temb fp32 [T, w]; NULL: nothing), then h bf16 [rows, w] = LN(x[r]).  w a multiple of 128, <= 1024. */
int b200_debug_temporal_embed_ln(int device, float* x, const float* temb, int N, int T, const float* gamma,
                                 const float* beta, float eps, int rows, int w, void* h, void* stream);
/* Attention over the T frames (1..16) of every (video, token) pair: qkv bf16 [n*T*N, 3W] (q | k | v, rows (b T + t) N
 * + token), heads of 64 (W = 64 H), no mask, scale 1/8 -> out bf16 [n*T*N, W] in the same row order. */
int b200_debug_temporal_attention(int device, const void* qkv, int n, int T, int N, int W, int H, void* out,
                                  void* stream);
/* Mean device time (ms, CUDA events) of `iters` back-to-back temporal_attention launches on device-generated data. */
int b200_debug_temporal_attention_time(int device, int n, int T, int N, int W, int H, int iters, float* out_ms);
/* LanguageBind's video transform of uint8 RGB frames [frames, h, w, 3] -> out fp32 CHW [frames, 3, S, S] (see
 * b200_model_encode_videos_u8); mean3 / std3 host fp32 [3]. */
int b200_debug_video_resize_crop(int device, const uint8_t* frames_hwc, int frames, int h, int w, int S,
                                 const float* mean3, const float* std3, float* out, void* stream);
/* out fp32 [n, E] = src / |src| per row if normalize, else src. */
int b200_debug_l2_rows(int device, const float* src, int n, int E, int normalize, float* out, void* stream);
/* ResNet stem im2col: exactly one of hwc (uint8 [n,S,S,3], normalised with mean3 / std3, host fp32 [3]) and chw (fp32
 * [n,3,S,S]) -> out bf16 [n*(S/2)^2, 64]. */
int b200_debug_stem_im2col(int device, const uint8_t* hwc, const float* chw, int n, int S, const float* mean3,
                           const float* std3, void* out, void* stream);
/* AvgPool2d(2) over NHWC x bf16 [n,H,W,C] -> out bf16 [n,H/2,W/2,C]. */
int b200_debug_avgpool2(int device, const void* x, int n, int H, int W, int C, void* out, void* stream);
/* ResNet attention-pool tokens: x bf16 [n,HW,C], pos fp32 [HW+1, C] -> out bf16 [n*(HW+1), C]: row 0 = mean_s x_s +
 * pos[0], row 1+s = x_s + pos[1+s]. */
int b200_debug_attnpool_tokens(int device, const void* x, const float* pos, int n, int HW, int C, void* out,
                               void* stream);
/* ViT im2col of fp32 CHW [n,3,S,S] -> out bf16 [n*((S/p)^2 + cls), kpad], k = c*p*p + dy*p + dx. */
int b200_debug_im2col_f32(int device, const float* chw, int n, int S, int p, int kpad, int cls, void* out, void* stream);
/* The JPEG decoder's arithmetic (shared __host__ __device__ code of the two kernels) run on the host: lets the CPU test
 * suite pin it against Pillow pixel for pixel.  A test hook, not a product path.  out_rgb == NULL: size query. */
int b200_debug_jpeg_decode_host(const uint8_t* file, size_t nbytes, uint8_t* out_rgb, size_t out_capacity,
                                int32_t* out_height, int32_t* out_width);
/* Pillow-compatible bicubic resize (shortest side -> S) + centre crop of uint8 HWC images [n,h,w,3] -> [n,S,S,3]. */
int b200_debug_resize(int device, const uint8_t* hwc, int n, int h, int w, int S, uint8_t* out, void* stream);
/* The same bicubic resampling squashed to S x S (x and y scaled independently, no crop): PIL resize((S, S), BICUBIC),
 * SigLIP's preprocessing. */
int b200_debug_resize_squash(int device, const uint8_t* hwc, int n, int h, int w, int S, uint8_t* out, void* stream);
/* The resize of n images of any sizes in one pass, as b200_model_encode_images_u8_ragged runs it: image i is uint8 HWC
 * [heights[i], widths[i], 3] at device pointer d_hwc[i] (d_hwc, heights and widths are host arrays) -> out
 * [n, S, S, 3]; squash 0: shortest side -> S + centre crop, as b200_debug_resize; squash 1: as
 * b200_debug_resize_squash. */
int b200_debug_resize_ragged(int device, const uint8_t* const* d_hwc, const int32_t* heights, const int32_t* widths,
                             int n, int S, int squash, uint8_t* out, void* stream);
/* Single-query attention pooling: for image b and head h, softmax(q_h . k_{b,s} / sqrt(D)) over the S tokens of image
 * b, times v_{b,s}, D = W / H.  q fp32, image b's query at q + b * q_stride: q_stride 0 shares one latent query [W] by
 * every image (SigLIP's MAP head, CoCa's pooler), q_stride W gives one per image [B, W] (the ResNet attention pool).
 * kv bf16 [B*S, 2W] (K columns then V columns); head_dim D 64 or 96.  out bf16 [B, W]. */
int b200_debug_map_attention(int device, const float* q, int q_stride, const void* kv, int B, int S, int W, int H,
                             void* out, void* stream);
/* One convolution of the ResNet CLIP image tower, on the path the model runs it: out bf16 = act(conv(x) + bias
 * (+ residual)).  w is a host array fp32 [cout, cin, k, k] (torch layout), laid out and rounded to bf16 as the model's
 * finalize does; bias fp32 [cout].  cin == 3: the stem conv1 (k 3, stride 2, padding 1) of x fp32 CHW [n, 3, H, W],
 * already normalised, as b200_model_encode_images_f32 receives it; out [n, H/2, W/2, cout].  Otherwise x bf16 NHWC
 * [n, H, W, cin] and k 1 (a GEMM over the pixels) or 3 (the implicit GEMM, stride 1, padding 1, cin a power of two
 * >= 32); out [n, H, W, cout].  relu != 0: ReLU, with the optional residual bf16 [n, H, W, cout] added before it;
 * relu == 0 (1 x 1 and stem convs only) takes no residual. */
int b200_debug_conv2d(int device, const void* x, int n, int H, int W, int cin, const float* w, int cout, int k,
                      const float* bias, const void* residual, int relu, void* out, void* stream);
/* ConvNeXt block head: x fp32 NHWC [n, H, W, C] -> out bf16 [n*H*W, C] = LayerNorm over C (gamma, beta, eps) of the
 * 7 x 7 depthwise conv with zero padding 3 plus bias; w fp32 [49, C], tap 7 dy + dx major (conv_dw.weight [C, 1, 7, 7]
 * transposed).  C a multiple of 64, <= 3072. */
int b200_debug_dwconv7_ln(int device, const float* x, int n, int H, int W, int C, const float* w, const float* bias,
                          const float* gamma, const float* beta, float eps, void* out, void* stream);
/* ConvNeXt per-pixel LayerNorm of x fp32 NHWC [n, H, W, C].  patchify 0: out fp32 [n*H*W, C] (may be x), the stem's
 * norm; patchify 1 (H, W even): out bf16 [n*(H/2)*(W/2), 4C], the downsample conv's GEMM rows, pixel (y, x) at column
 * ((y % 2) * 2 + x % 2) * C + c of row (y/2, x/2).  C a multiple of 64, <= 3072. */
int b200_debug_ln_pixels(int device, const float* x, int n, int H, int W, int C, const float* gamma, const float* beta,
                         float eps, int patchify, void* out, void* stream);
/* ConvNeXt head input: mean over the HW pixel rows of each image of x fp32 [n, HW, C], then LayerNorm -> out bf16
 * [n, C].  C a multiple of 64, <= 3072. */
int b200_debug_pool_ln(int device, const float* x, int n, int HW, int C, const float* gamma, const float* beta, float eps,
                       void* out, void* stream);
/* Transformer layers [first, first + count) of a finalized model's vision (tower 0) or text (tower 1) tower, through
 * the layer runner the encode calls use, with the tower's own mask: none for vision and SigLIP text, causal for CLIP
 * text (CoCa's too: its CLS row's keys follow ids this hook does not take), key lengths for the BERT family, MPNet,
 * XLM-R and GTE.  x_in fp32 [B*S, width] is the residual stream the first layer reads (a post-LN tower also gets
 * h = bf16(x_in), as its embedding LayerNorm leaves them); kv_len int32 [B] (NULL: S for every sequence), each in 0..S, is read by the key-length towers only.  S must be the vision
 * tower's token count, or 1..ctx for a text tower.  The call first waits for the model's own stream (an encode call
 * with sync = 0 may still use the workspaces), then runs on `stream`.  Afterwards, each output that is not NULL
 * receives what the last layer left: x_out fp32 [B*S, width] the residual stream; h_out bf16 [B*S, width] the last
 * LayerNorm output (pre-LN: bf16(LN2(x_mid)), fc1's input; post-LN: bf16(x_out)); qkv_out bf16 [B*S, 3*aw] the QKV
 * projection after any rotary embedding; o_out bf16 [B*S, aw] the attention output; u_out bf16 [B*S, fc1] the MLP
 * hidden rows after the activation or gate (a gated MLP's result in the first fc1 / 2 columns).  width, aw and fc1
 * come from b200_debug_layer_cols.  Nothing but the model's workspaces and the outputs is written.
 * B200_ERR_INVALID_ARG for a tower the model lacks, a range outside the tower, B above max_batch, B*S above the
 * workspace, a bad S or a key length outside 0..S. */
int b200_debug_layers(b200_model* m, int tower, int first, int count, const float* x_in, int B, int S,
                      const int32_t* kv_len, float* x_out, void* h_out, void* qkv_out, void* o_out, void* u_out,
                      void* stream);
/* The row widths of b200_debug_layers' outputs for a finalized model's tower: out[0] the width, out[1] aw (heads times
 * the attention kernel's head dim: the tower's, or 96 for 80 and 88 and 128 for 104, zero-padded), out[2] fc1 (mlp, or
 * for a gated MLP both halves of mlp rounded up to 64).  out: host int32 [3].  B200_ERR_INVALID_ARG for a tower the
 * model lacks. */
int b200_debug_layer_cols(b200_model* m, int tower, int32_t* out);
/* Bytes of device memory the library holds right now, over all devices and handles of this process (indexes,
 * exchanges, models and the scratch of calls in flight).  Memory from b200_host_alloc is not counted.  Returns to its
 * earlier value once every handle created in between is destroyed: a leak check. */
int b200_debug_device_bytes(int64_t* out_live_bytes);

#ifdef __cplusplus
}
#endif
#endif /* MARQO_B200_H */
