// Encoder runtime: CLIP ViT image tower, CLIP text tower, SigLIP towers, OpenAI ResNet CLIP, ConvNeXt CLIP, EVA02
// CLIP and CoCa image towers, CoCa's text tower, BERT (e5,
// MiniLM, bge), MPNet, XLM-R (multilingual-e5), GTE (Stella) — SURVEY §8 a2-a5.
//
// What the reference calls (third-party, restated in oracle/encoders.py):
//   OPEN_CLIP.encode_image / encode_text   src/marqo/core/inference/embedding_models/open_clip_model.py:249-286
//   HuggingFaceModel.encode                src/marqo/core/inference/embedding_models/hugging_face_model.py:172-214
//
// Data layout in HBM (per model handle):
//   weights   bf16 [out, in] for every Linear (wgmma B operand, K-major), fp32 for LayerNorm / biases /
//             embeddings / projections
//   x         fp32 [tokens, width]   residual stream (kept fp32 end to end)
//   h         bf16 [tokens, width]   LayerNorm output = GEMM A operand
//   qkv       bf16 [tokens, 3*aw]    fused QKV projection (aw: TowerW::aw, the width with zero-padded heads)
//   o         bf16 [tokens, aw]      attention output
//   u         bf16 [tokens, fc1_cols] MLP hidden: mlp columns, or both halves of a gated MLP (2 mlp, see Mlp)
//   patches   bf16 [images * (grid^2 + 1), kpad]  im2col of preprocessed fp32 CHW input (zero class-token rows)
// Every Linear is the wgmma GEMM of gemm.cu with bias / activation / residual-add fused into its epilogue.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <map>
#include <tuple>
#include <mutex>
#include <string>
#include <vector>

#include "attention.cuh"
#include "common.cuh"
#include "gemm.cuh"
#include "kernels.cuh"

using namespace mb;

namespace {

struct LayerW {
    const float *ln1_w = nullptr, *ln1_b = nullptr, *ln2_w = nullptr, *ln2_b = nullptr;
    const float *b_qkv = nullptr, *b_o = nullptr, *b_fc = nullptr, *b_proj = nullptr;
    const __nv_bfloat16 *w_qkv = nullptr, *w_o = nullptr, *w_fc = nullptr, *w_proj = nullptr;
    // EVA02: attn.norm over the attention output [width] and mlp.norm over the SwiGLU hidden row [TowerW::mlp_h]
    const float *ln_attn_w = nullptr, *ln_attn_b = nullptr, *ln_mlp_w = nullptr, *ln_mlp_b = nullptr;
    // LanguageBind's temporal step (TowerW::frames > 0): temporal_embedding [frames, width] (NULL for one frame, which
    // adds none), temporal_layer_norm1, temporal_attn's fused q | k | v [3 width, width] and out_proj
    const float *temb = nullptr, *tln_w = nullptr, *tln_b = nullptr, *b_tqkv = nullptr, *b_to = nullptr;
    const __nv_bfloat16 *w_tqkv = nullptr, *w_to = nullptr;
};

// A layer's MLP: fc1 with the tower's activation in its epilogue, or a gated unit over the 2 mlp columns fc1 writes
// without one (EVA02's SwiGLU with its LayerNorm, GTE's GeGLU), run in place over one half, which fc2 reads at row
// stride 2 mlp.
enum class Mlp { ACT, SWIGLU_LN, GEGLU };

// SigLIP's MAP pooling head (timm AttentionPoolLatent with one latent): q = latent W_q^T + b_q is batch-independent and
// built once by b200_model_finalize.  CoCa's attentional pooler uses q (ln_q(query[0]) W_q^T + b_q, [embed_dim]), w_kv /
// b_kv (k_proj | v_proj, [2 embed_dim, width]), w_proj / b_proj (out_proj) and ln_w / ln_b (ln_k, [width]).
struct MapW {
    const float* q = nullptr;                                    // fp32 [width]
    const __nv_bfloat16 *w_kv = nullptr, *w_proj = nullptr, *w_fc1 = nullptr, *w_fc2 = nullptr;
    const float *b_kv = nullptr, *b_proj = nullptr, *b_fc1 = nullptr, *b_fc2 = nullptr, *ln_w = nullptr, *ln_b = nullptr;
    int mlp = 0;
};

// What runs a tower, resolved once from the model's arch (resolve_kinds).  Archs whose forward passes differ only in
// data share a kind: MPNet and XLM-R are ROBERTA, and the ResNet CLIP's text tower is CLIP's.
enum class VisionKind { NONE, CLIP_VIT, SIGLIP_VIT, RESNET, CONVNEXT, EVA_VIT, COCA_VIT, VIDEO_VIT };
enum class TextKind { NONE, CLIP, SIGLIP, BERT, ROBERTA, GTE, COCA };
struct Kinds {
    VisionKind vision = VisionKind::NONE;
    TextKind text = TextKind::NONE;
    bool mpnet = false;   // ROBERTA: MPNet's layer names and relative-position bias, else XLM-R's token-type row
};

// The model calls of the C ABI by what they run, which decides whether a model takes them (require_accepts): IMAGES
// every image encode (u8, u8 device, ragged, ragged device, f32), TOKENS encode_tokens(_device), CLASSIFY
// classify_tokens(_device), DETECT detect_images_u8, VIDEOS encode_videos_u8(_device).
enum class Call { IMAGES, TOKENS, CLASSIFY, DETECT, VIDEOS };

struct TowerW {
    b200_tower_desc d{};
    // the attention width heads * kernel_head_dim(width / heads): width, or for the ViT-H / g / bigG vision towers the
    // width with every head zero-padded to the kernel's head dim (pad_heads)
    int aw = 0;
    std::vector<LayerW> layers;
    float eps = 1e-5f;                      // every LayerNorm of the tower
    // pre-LN layers (open_clip, timm) normalise before attention and the MLP; post-LN ones (BERT family, GTE) after
    bool pre_ln = true;
    Mlp mlp_form = Mlp::ACT;
    int act = gemm::ACT_GELU;               // Mlp::ACT: the activation in fc1's epilogue
    // the MLP's hidden size; T.d.mlp, the width its GEMMs run, is EVA02's rounded up to 64
    int mlp_h = 0;
    // RoPE on q and k after the QKV GEMM (kernels::rope_qk): fp32 (cos, sin) pairs, EVA02's [grid^2, 32]
    // (kernels::rope_table), GTE's [ctx, 32] (kernels::rope_table_ntk); the rows before rope_first of every sequence
    // (EVA02's class row) are not rotated
    const float* rope = nullptr;
    kernels::RopePairing rope_pairing = kernels::RopePairing::INTERLEAVED;
    int rope_first = 0;
    // tokens per item: an image's token rows, or the longest sequence (a video tower: one frame's)
    int tokens = 0;
    // LanguageBind's video tower: frames per video (0: not a video tower), and the factor exp(logit_scale) of its head
    int frames = 0;
    float out_scale = 1.f;
    // vision
    const __nv_bfloat16* conv_w = nullptr;  // [width, kpad]
    const __nv_bfloat16* conv_wg = nullptr; // [width, gemm::patch_gather_k(patch)]: gather GEMM order
    int kpad = 0, grid = 0;
    int cls_rows = 1;                       // class-token rows per image: 1 (CLIP), 0 (SigLIP)
    // pos: CLIP positional_embedding [grid^2 + 1, width]; SigLIP pos_embed + the patch conv's bias [grid^2, width].
    // ln_pre is NULL for SigLIP.
    const float *cls = nullptr, *pos = nullptr, *ln_pre_w = nullptr, *ln_pre_b = nullptr;
    // final LN (ln_post / ln_final / trunk.norm) and CLIP's projection [width, embed] (M-CLIP's text head: its
    // LinearTransformation transposed, with b_tproj its bias)
    const float *ln_out_w = nullptr, *ln_out_b = nullptr, *proj = nullptr;
    // SigLIP text projection and EVA02's vision head (nn.Linear [embed, width] + bias); SigLIP's vision MAP head and
    // CoCa's attentional pooler
    const __nv_bfloat16* w_tproj = nullptr;
    const float* b_tproj = nullptr;
    MapW map;
    // text / bert embeddings; CoCa's text cls_emb [width]
    const float *tok = nullptr, *type0 = nullptr, *emb_ln_w = nullptr, *emb_ln_b = nullptr, *text_cls = nullptr;
    // MPNet: relative-position bias of every layer, fp32 [heads, 2 * ctx - 1] pre-scaled by log2(e)
    attention::RelBias rel_bias;
    // BertForSequenceClassification (cls_labels > 0): the pooler [width, width] and [width], the classifier
    // [cls_labels, width] and [cls_labels], all fp32 as uploaded
    const float *pool_w = nullptr, *pool_b = nullptr, *cls_w = nullptr, *cls_b = nullptr;
};

// OpenAI ResNet CLIP image tower (open_clip ModifiedResNet, verify): every conv with its BatchNorm folded in at
// finalize (w' = w g / sqrt(var + eps), b' = beta - mean g / sqrt(var + eps), in double), in the k order of the kernel
// that runs it (gemm::conv_rows_k).
struct ConvW {
    const __nv_bfloat16* w = nullptr;   // bf16 [cout, conv_rows_k(cin, k)]
    const float* b = nullptr;           // fp32 [cout]
    int cin = 0, cout = 0, k = 0;
};

struct BottleneckW {
    ConvW c1, c2, c3, ds;   // ds: the downsample conv (has_ds)
    int stride = 1;
    bool has_ds = false;
};

// Activations are NHWC bf16 in four buffers of max_batch * per_image elements, which the forward pass rotates through
// (forward_resnet); fixed pointers, so captured CUDA graphs replay them.
struct ResnetW {
    ConvW stem[3];
    std::vector<BottleneckW> blocks;
    int C = 0, grid = 0;                 // trunk output channels and side
    const float* pos = nullptr;          // attnpool.positional_embedding [grid^2 + 1, C]
    const __nv_bfloat16 *w_kv = nullptr, *w_q = nullptr, *w_c = nullptr;   // [2C, C] (k_proj | v_proj), [C, C], [E, C]
    const float *b_kv = nullptr, *b_q = nullptr, *b_c = nullptr;
    DeviceBuffer<__nv_bfloat16> buf[4];
};

// ConvNeXt CLIP image tower (open_clip TimmModel over timm's ConvNeXt, verify).  Its stem conv is the ViT patch
// embedding at patch 4 without class rows (TowerW conv_w / conv_wg of m->vision).  A block is the MLP half of a pre-LN
// transformer layer behind a depthwise conv: dwconv7_ln -> h, fc1 (+ GELU) -> u, fc2 with gamma folded into its rows
// and bias, added onto the fp32 residual stream x in place.
struct ConvnextBlockW {
    const float *dw_w = nullptr, *dw_b = nullptr;   // fp32 [49, C] (tap-major), [C]
    const float *ln_w = nullptr, *ln_b = nullptr, *b1 = nullptr, *b2 = nullptr;
    const __nv_bfloat16 *w1 = nullptr, *w2 = nullptr;   // [4C, C], gamma-scaled [C, 4C]
};

struct ConvnextStageW {
    int C = 0;
    // downsample (stages > 0): LayerNorm, then the 2 x 2 stride-2 conv as a GEMM over ln_pixels' patch rows
    const float *ds_ln_w = nullptr, *ds_ln_b = nullptr, *ds_b = nullptr;
    const __nv_bfloat16* ds_w = nullptr;   // [C, 4 C_prev], column (dy * 2 + dx) * C_prev + c
    std::vector<ConvnextBlockW> blocks;
};

// The activations live in x / h / u of max_images images at the first stage, the largest (every later stage has a
// quarter of the pixels and twice the channels); fixed pointers, so captured CUDA graphs replay them.
struct ConvnextW {
    ConvnextStageW stages[4];
    const float *stem_b = nullptr, *stem_ln_w = nullptr, *stem_ln_b = nullptr;
    const float *head_ln_w = nullptr, *head_ln_b = nullptr;
    const __nv_bfloat16* w_proj = nullptr;                              // linear head [E, C3]
    const __nv_bfloat16 *w_fc1 = nullptr, *w_fc2 = nullptr;             // MLP head [2E, C3], [E, 2E]
    const float* b_fc1 = nullptr;
    int max_images = 0;
    DeviceBuffer<float> x;                 // [pixels, C]
    DeviceBuffer<__nv_bfloat16> h, u;      // [pixels, C], [pixels, 4C]
};

// OWL-ViT's detection head (owl_detect): the detector's LayerNorm; the class head as one Linear [ncls, width] whose
// rows are class_head.dense0 (embed_dim rows), logit_shift, logit_scale and zero rows up to a multiple of 64, with its
// fp32 bias; box_head.dense0 / dense1 (bf16, GELU in their epilogues) and dense2 (fp32 [4, width], owl_boxes); the
// box bias table fp32 [G^2, 4].
struct OwlW {
    const float *ln_w = nullptr, *ln_b = nullptr, *b_cls = nullptr, *b_box0 = nullptr, *b_box1 = nullptr;
    const float *w_box2 = nullptr, *b_box2 = nullptr, *box_bias = nullptr;
    const __nv_bfloat16 *w_cls = nullptr, *w_box0 = nullptr, *w_box1 = nullptr;
    int ncls = 0;
};

}  // namespace

struct b200_model {
    int device = 0;
    int sms = 0;
    b200_model_desc desc{};
    bool finalized = false;
    std::map<std::string, DeviceBuffer<float>> raw;   // uploaded fp32 parameters by checkpoint name
    std::vector<DeviceBuffer<uint8_t>> derived;        // device buffers built from them by b200_model_finalize
    Kinds kind;
    TowerW vision, text;
    ResnetW resnet;   // VisionKind::RESNET's image tower (vision.tokens = grid^2 + 1)
    ConvnextW convnext;   // VisionKind::CONVNEXT's image tower (vision.tokens = the stem's (S/4)^2 pixels)
    OwlW owl;             // owl_detect's head
    DeviceBuffer<float> det;   // owl_detect: [max_batch, G^2] logits, then [max_batch, G^2, 4] boxes
    // workspaces (sized for max_tokens tokens)
    long long max_tokens = 0;
    DeviceBuffer<float> x;
    DeviceBuffer<__nv_bfloat16> h, qkv, o, u, patches;
    DeviceBuffer<int32_t> aux;        // [max_batch] eot index / kv_len
    DeviceBuffer<float> out_dev;      // [max_batch, embed]
    DeviceBuffer<float> pooled;       // [max_batch, width] LayerNorm-ed pooled rows (CLIP heads)
    DeviceBuffer<uint8_t> in_dev;     // staging for host inputs
    DeviceBuffer<uint8_t> resized;    // [max_batch, S, S, 3]
    DeviceBuffer<float> video_f32;    // a video model's transformed frames: fp32 CHW [videos per pass * frames, 3, S, S]
    cudaStream_t stream = nullptr;
    UniqueStream own_stream;          // created by the handle; `stream` may be replaced by a caller's stream
    UniqueEvent ev0, ev1;
    bool timing_valid = false;
    int last_launches = 0;
    // optional per-kernel-class device timing (bench.py's roofline numerator)
    bool profiling = false;
    std::vector<UniqueEvent> prof_ev;  // pairs
    std::vector<int> prof_cls;         // 0 = gemm, 1 = attention
    int prof_n = 0;
    // CUDA graphs of small (launch-bound) forward passes, keyed by everything the captured launches depend on
    struct GraphKey {
        Call pass;   // forward_images (IMAGES), forward_tokens (TOKENS), forward_detect or forward_videos
        int n, S, normalize;
        const void *in0, *in1, *out;
        const void* in2 = nullptr;   // token-type ids of a classified pair batch
        bool operator<(const GraphKey& o) const {
            return std::tie(pass, n, S, normalize, in0, in1, out, in2) <
                   std::tie(o.pass, o.n, o.S, o.normalize, o.in0, o.in1, o.out, o.in2);
        }
    };
    struct GraphEntry {
        UniqueGraphExec exec;   // null: seen once (ran eagerly), captured on the next use
        int launches = 0;
    };
    std::map<GraphKey, GraphEntry> graphs;
    bool external_stream = false;
    std::mutex mu;
};

namespace {

// A device buffer built from the checkpoint, owned by the model until it is destroyed.
template <class T>
T* derived_buffer(b200_model* m, size_t n) {
    m->derived.emplace_back(n * sizeof(T));
    return reinterpret_cast<T*>(m->derived.back().get());
}

// The attention kernels' head dim for a tower's head dim hd: hd itself for 32 and 64; 80 and 88 run as 96 and 104 as
// 128, each head padded with zero columns (pad_heads).
int kernel_head_dim(int hd) { return hd <= 64 ? hd : hd <= 96 ? 96 : 128; }

// max_width: 1664 for the CLIP towers (their LayerNorm and head kernels), 1024 for the others.  padded_heads: the tower
// may have head dims 80, 88 and 104, which only the wgmma attention kernel runs (kernel_head_dim), so only a vision
// tower of at least 128 tokens takes them.
void check_tower(const b200_tower_desc& t, const char* name, int max_width = 1024, bool padded_heads = false) {
    MB_CHECK_ARG(t.width > 0 && t.width % 128 == 0 && t.width <= max_width, "%s.width %d must be a multiple of 128, <= %d",
                 name, t.width, max_width);
    MB_CHECK_ARG(t.layers > 0, "%s.layers must be positive", name);
    const int hd = t.heads > 0 && t.width % t.heads == 0 ? t.width / t.heads : 0;
    const bool padded = padded_heads && (hd == 80 || hd == 88 || hd == 104);
    MB_CHECK_ARG(hd == 32 || hd == 64 || padded, "%s: head_dim must be 32 or 64%s (width %d, heads %d)", name,
                 padded_heads ? ", or 80, 88 or 104" : "", t.width, t.heads);
    MB_CHECK_ARG(t.mlp > 0 && t.mlp % 64 == 0, "%s.mlp %d must be a multiple of 64", name, t.mlp);
}

// The only reader of desc.arch besides b200_model_create's unknown-arch check.
Kinds resolve_kinds(const b200_model_desc& d) {
    Kinds k;
    const bool vit = d.vision.layers > 0, text = d.text.layers > 0;
    switch (d.arch) {
    case B200_ARCH_CLIP:
        if (vit)
            k.vision = d.attn_pool_heads > 0 ? VisionKind::COCA_VIT
                       : d.video_frames > 0  ? VisionKind::VIDEO_VIT
                                             : VisionKind::CLIP_VIT;
        if (text) k.text = d.text_embed_cls ? TextKind::COCA : TextKind::CLIP;
        break;
    case B200_ARCH_CLIP_RESNET:
        if (d.resnet_layers[0] > 0) k.vision = VisionKind::RESNET;
        if (text) k.text = TextKind::CLIP;
        break;
    case B200_ARCH_CLIP_CONVNEXT:
        if (d.convnext_depths[0] > 0) k.vision = VisionKind::CONVNEXT;
        if (text) k.text = TextKind::CLIP;
        break;
    case B200_ARCH_CLIP_EVA:
        if (vit) k.vision = VisionKind::EVA_VIT;
        if (text) k.text = TextKind::CLIP;
        break;
    case B200_ARCH_SIGLIP:
        if (vit) k.vision = VisionKind::SIGLIP_VIT;
        if (text) k.text = TextKind::SIGLIP;
        break;
    case B200_ARCH_BERT:
        if (text) k.text = TextKind::BERT;
        break;
    case B200_ARCH_MPNET:
    case B200_ARCH_XLMR:
        if (text) k.text = TextKind::ROBERTA;
        k.mpnet = d.arch == B200_ARCH_MPNET;
        break;
    case B200_ARCH_GTE:
        if (text) k.text = TextKind::GTE;
        break;
    }
    return k;
}

// the model-wide settings of a SigLIP tower
void check_siglip(const b200_model_desc& d) {
    MB_CHECK_ARG(d.layer_norm_eps > 0.f, "SigLIP: layer_norm_eps must be positive");
    MB_CHECK_ARG(d.embed_dim % 32 == 0, "SigLIP: embed_dim %d must be a multiple of 32", d.embed_dim);
}

void check_vision(const b200_model_desc& d, VisionKind kind) {
    if (kind == VisionKind::NONE) return;
    for (int i = 0; i < 3; ++i) MB_CHECK_ARG(d.image_std[i] > 0.f, "image_std must be positive");
    switch (kind) {
    case VisionKind::RESNET: {
        const int wd = d.resnet_width, S = d.resnet_image_size;
        for (int s = 0; s < 4; ++s)
            MB_CHECK_ARG(d.resnet_layers[s] > 0 && d.resnet_layers[s] <= 64, "resnet_layers[%d] = %d out of range", s,
                         d.resnet_layers[s]);
        // the stem's 3 x 3 convs gather width / 2 channels and write width / 2 columns: a multiple of 8
        MB_CHECK_ARG(wd >= 64 && wd <= 128 && wd % 16 == 0, "resnet_width %d must be a multiple of 16 in [64, 128]", wd);
        MB_CHECK_ARG(S > 0 && S % 32 == 0 && S <= 512, "resnet_image_size %d must be a multiple of 32, <= 512", S);
        MB_CHECK_ARG(d.resnet_heads * 64 == 32 * wd, "attention pool: head_dim must be 64 (%d channels, %d heads)",
                     32 * wd, d.resnet_heads);
        MB_CHECK_ARG(d.embed_dim % 32 == 0, "CLIP ResNet: embed_dim %d must be a multiple of 32", d.embed_dim);
        break;
    }
    case VisionKind::CONVNEXT: {
        // the per-pixel kernels take multiples of 64 channels up to 3072; the image halves four times after the stem
        for (int s = 0; s < 4; ++s) {
            MB_CHECK_ARG(d.convnext_dims[s] > 0 && d.convnext_dims[s] % 64 == 0 && d.convnext_dims[s] <= 3072,
                         "convnext_dims[%d] = %d must be a multiple of 64, <= 3072", s, d.convnext_dims[s]);
            MB_CHECK_ARG(d.convnext_depths[s] > 0 && d.convnext_depths[s] <= 64, "convnext_depths[%d] = %d out of range",
                         s, d.convnext_depths[s]);
        }
        const int S = d.convnext_image_size;
        MB_CHECK_ARG(S > 0 && S % 32 == 0 && S <= 640, "convnext_image_size %d must be a multiple of 32, <= 640", S);
        MB_CHECK_ARG(d.convnext_head == 0 || d.convnext_head == 1, "convnext_head %d must be 0 (linear) or 1 (MLP)",
                     d.convnext_head);
        MB_CHECK_ARG(d.embed_dim % 32 == 0, "CLIP ConvNeXt: embed_dim %d must be a multiple of 32", d.embed_dim);
        MB_CHECK_ARG(d.layer_norm_eps > 0.f, "CLIP ConvNeXt: layer_norm_eps must be positive");
        break;
    }
    case VisionKind::EVA_VIT: {
        // heads of 64 (the RoPE pairs), widths up to 1024, and a SwiGLU hidden size of any value whose round-up to 64
        // swiglu_ln holds; the GEMMs run it padded (build_eva_vision)
        MB_CHECK_ARG(d.vision.patch > 0 && d.vision.image_size % d.vision.patch == 0,
                     "image_size must be a multiple of patch");
        MB_CHECK_ARG(d.vision.mlp > 0 && (int)round_up((size_t)d.vision.mlp, 64) <= kernels::SWIGLU_MAX_HP,
                     "EVA02: vision.mlp %d must be positive and round up to at most %d", d.vision.mlp,
                     kernels::SWIGLU_MAX_HP);
        b200_tower_desc t = d.vision;
        t.mlp = (int)round_up((size_t)t.mlp, 64);
        check_tower(t, "vision");
        MB_CHECK_ARG(d.vision.width == d.vision.heads * 64, "EVA02: vision head_dim must be 64 (width %d, heads %d)",
                     d.vision.width, d.vision.heads);
        MB_CHECK_ARG(d.layer_norm_eps > 0.f, "EVA02: layer_norm_eps must be positive");
        MB_CHECK_ARG(d.eva_rope_ref_grid > 0, "EVA02: eva_rope_ref_grid %d must be positive", d.eva_rope_ref_grid);
        MB_CHECK_ARG(d.embed_dim % 32 == 0, "EVA02: embed_dim %d must be a multiple of 32", d.embed_dim);
        break;
    }
    case VisionKind::SIGLIP_VIT:
        check_siglip(d);
        // the MAP head has no projection; its single-query attention runs head_dim 64 only
        MB_CHECK_ARG(d.embed_dim == d.vision.width, "SigLIP: embed_dim %d must equal the vision width %d", d.embed_dim,
                     d.vision.width);
        MB_CHECK_ARG(d.vision.width == d.vision.heads * 64, "SigLIP: vision head_dim must be 64 (width %d, heads %d)",
                     d.vision.width, d.vision.heads);
        [[fallthrough]];
    case VisionKind::COCA_VIT:
        if (kind == VisionKind::COCA_VIT) {
            // the pooler's single-query attention runs head dims 64 and 96; its K|V rows and output fit the trunk's
            // qkv and o workspaces
            const int ph = d.attn_pool_heads, pd = ph > 0 && d.embed_dim % ph == 0 ? d.embed_dim / ph : 0;
            MB_CHECK_ARG(pd == 64 || pd == 96, "CoCa: attn_pool_heads %d must give embed_dim %d a head dim of 64 or 96",
                         ph, d.embed_dim);
            MB_CHECK_ARG(d.embed_dim <= d.vision.width, "CoCa: embed_dim %d must be at most the vision width %d",
                         d.embed_dim, d.vision.width);
        }
        [[fallthrough]];
    case VisionKind::VIDEO_VIT:
        if (kind == VisionKind::VIDEO_VIT) {
            // the temporal kernels: heads of 64, the LayerNorm's rows of up to 1024 in registers
            MB_CHECK_ARG(d.vision.width == d.vision.heads * 64 && d.vision.width <= 1024,
                         "video: vision head_dim must be 64 and width <= 1024 (width %d, heads %d)", d.vision.width,
                         d.vision.heads);
        }
        [[fallthrough]];
    case VisionKind::CLIP_VIT: {
        MB_CHECK_ARG(d.vision.patch > 0 && d.vision.image_size % d.vision.patch == 0,
                     "image_size must be a multiple of patch");
        const bool clip = kind == VisionKind::CLIP_VIT || kind == VisionKind::COCA_VIT || kind == VisionKind::VIDEO_VIT;
        const int grid = d.vision.image_size / d.vision.patch;
        check_tower(d.vision, "vision", clip ? 1664 : 1024, clip && grid * grid + 1 >= 128);
        break;
    }
    }
    MB_CHECK_ARG(d.resize_squash == 0 || d.resize_squash == 1, "resize_squash %d must be 0 or 1", d.resize_squash);
}

// OWL-ViT's detector: the CLIP ViT and text towers, squashed images, the merge LayerNorm's width limit, and a class
// head of embed_dim + 2 rows padded to 64 whose fp32 output fits the trunk's residual rows
void check_owl(const b200_model_desc& d, const Kinds& k) {
    MB_CHECK_ARG(d.owl_detect == 0 || d.owl_detect == 1, "owl_detect %d must be 0 or 1", d.owl_detect);
    if (!d.owl_detect) return;
    MB_CHECK_ARG(d.arch == B200_ARCH_CLIP, "owl_detect: only the CLIP arch takes OWL-ViT's detection head");
    MB_CHECK_ARG(k.vision == VisionKind::CLIP_VIT && k.text == TextKind::CLIP,
                 "owl_detect: the detector needs the CLIP ViT vision tower and the CLIP text tower");
    MB_CHECK_ARG(d.resize_squash == 1, "owl_detect: OWL-ViT squashes its images (resize_squash 1)");
    MB_CHECK_ARG(d.vision.width <= 1024, "owl_detect: vision.width %d must be <= 1024", d.vision.width);
    MB_CHECK_ARG((int)round_up((size_t)d.embed_dim + 2, 64) <= d.vision.width,
                 "owl_detect: embed_dim %d + 2 rounded up to 64 must be at most vision.width %d", d.embed_dim,
                 d.vision.width);
}

// LanguageBind's video model: the CLIP ViT with the temporal step, its frame-mean head and the CLIP text tower
void check_video(const b200_model_desc& d, const Kinds& k) {
    MB_CHECK_ARG(d.video_frames >= 0 && d.video_frames <= kernels::TEMPORAL_MAX_FRAMES,
                 "video_frames %d must be 0..%d", d.video_frames, kernels::TEMPORAL_MAX_FRAMES);
    if (!d.video_frames) return;
    MB_CHECK_ARG(d.arch == B200_ARCH_CLIP, "video_frames: only the CLIP arch takes LanguageBind's video tower");
    MB_CHECK_ARG(d.attn_pool_heads == 0 && !d.owl_detect && !d.text_embed_cls,
                 "video_frames: CoCa's pooler and OWL-ViT's detector are other heads");
    MB_CHECK_ARG(k.vision == VisionKind::VIDEO_VIT, "video_frames: the model needs a vision tower");
}

void check_text(const b200_model_desc& d, const Kinds& k) {
    MB_CHECK_ARG(d.text_proj_dim >= 0, "text_proj_dim %d must not be negative", d.text_proj_dim);
    MB_CHECK_ARG(d.text_proj_dim == 0 || d.arch == B200_ARCH_BERT || d.arch == B200_ARCH_XLMR,
                 "text_proj_dim: only the BERT and XLM-R text towers take a projected head");
    MB_CHECK_ARG(d.cls_labels >= 0, "cls_labels %d must not be negative", d.cls_labels);
    MB_CHECK_ARG(d.cls_labels == 0 || d.arch == B200_ARCH_BERT,
                 "cls_labels: only the BERT arch takes a sequence-classification head");
    if (k.text == TextKind::NONE) return;
    check_tower(d.text, "text", k.text == TextKind::CLIP || k.text == TextKind::COCA ? 1664 : 1024);
    MB_CHECK_ARG(d.text.ctx > 0 && d.text.vocab > 0, "text.ctx and text.vocab must be positive");
    switch (k.text) {
    case TextKind::COCA:
        // the CLS mask lives in the mma.sync attention kernel (head_dim 64, fewer than 128 tokens)
        MB_CHECK_ARG(d.text.ctx >= 2 && d.text.ctx <= 127, "CoCa: text.ctx %d must be 2..127 with the CLS row",
                     d.text.ctx);
        MB_CHECK_ARG(d.text.width == d.text.heads * 64, "CoCa: text head_dim must be 64 (width %d, heads %d)",
                     d.text.width, d.text.heads);
        break;
    case TextKind::SIGLIP:
        check_siglip(d);
        break;
    case TextKind::ROBERTA: {
        const char* name = k.mpnet ? "MPNet" : "XLM-R";
        MB_CHECK_ARG(d.layer_norm_eps > 0.f, "%s: layer_norm_eps must be positive", name);
        MB_CHECK_ARG(d.pad_id >= 0 && d.pad_id < d.text.vocab, "%s: pad_id %d out of range", name, d.pad_id);
        if (k.mpnet) {
            MB_CHECK_ARG(d.text.width == d.text.heads * 64, "MPNet: head_dim must be 64 (width %d, heads %d)",
                         d.text.width, d.text.heads);
            MB_CHECK_ARG(d.rel_buckets >= 4 && d.rel_buckets % 2 == 0 && d.rel_max_distance > d.rel_buckets / 4,
                         "MPNet: bad relative-bias buckets (%d) / max distance (%d)", d.rel_buckets,
                         d.rel_max_distance);
            MB_CHECK_ARG(d.text.ctx <= 1024, "MPNet: sequences of up to 1024 tokens are supported (ctx %d)",
                         d.text.ctx);
        }
        [[fallthrough]];
    }
    case TextKind::BERT:
        if (d.cls_labels > 0) {
            // BertForSequenceClassification: the pooler and classifier (cls_head) write cls_labels scores per pair
            MB_CHECK_ARG(d.text_proj_dim == 0, "cls_labels and text_proj_dim are two different heads");
            MB_CHECK_ARG(d.embed_dim == d.cls_labels, "embed_dim %d must equal cls_labels %d", d.embed_dim,
                         d.cls_labels);
            break;
        }
        if (d.text_proj_dim > 0) {
            // M-CLIP's text head: the masked mean, projected (text_head)
            MB_CHECK_ARG(d.pool == B200_POOL_MEAN, "text_proj_dim: the projected head pools by the masked mean");
            MB_CHECK_ARG(d.embed_dim == d.text_proj_dim, "embed_dim %d must equal text_proj_dim %d", d.embed_dim,
                         d.text_proj_dim);
            break;
        }
        MB_CHECK_ARG(d.embed_dim == d.text.width, "BERT / MPNet / XLM-R embed_dim must equal width");
        break;
    case TextKind::GTE:
        // heads of 64 (the rotate-half pairs j, j + 32); the engine's sequences stop at 512 tokens
        MB_CHECK_ARG(d.text.width == d.text.heads * 64, "GTE: head_dim must be 64 (width %d, heads %d)", d.text.width,
                     d.text.heads);
        MB_CHECK_ARG(d.embed_dim == d.text.width, "GTE: embed_dim %d must equal width %d", d.embed_dim, d.text.width);
        MB_CHECK_ARG(d.text.ctx <= 512, "GTE: sequences of up to 512 tokens are supported (ctx %d)", d.text.ctx);
        MB_CHECK_ARG(d.layer_norm_eps > 0.f, "GTE: layer_norm_eps must be positive");
        MB_CHECK_ARG(d.rope_theta > 0.f && d.rope_ntk_factor >= 1.f,
                     "GTE: rope_theta (%g) must be positive and rope_ntk_factor (%g) at least 1", d.rope_theta,
                     d.rope_ntk_factor);
        break;
    }
}

const float* param(b200_model* m, const std::string& name, long long numel) {
    auto it = m->raw.find(name);
    if (it == m->raw.end()) fail(B200_ERR_MISSING_WEIGHT, "missing parameter '%s'", name.c_str());
    if ((long long)it->second.size() != numel)
        fail(B200_ERR_INVALID_ARG, "parameter '%s' has %zu elements, expected %lld", name.c_str(), it->second.size(),
             numel);
    return it->second.get();
}

// fp32 parameter -> owned bf16 copy; the fp32 original is released.
const __nv_bfloat16* to_bf16(b200_model* m, const std::string& name, long long numel) {
    const float* src = param(m, name, numel);
    __nv_bfloat16* dst = derived_buffer<__nv_bfloat16>(m, (size_t)numel);
    kernels::f32_to_bf16(src, dst, numel, m->stream);
    MB_CUDA(cudaStreamSynchronize(m->stream));
    m->raw.erase(name);
    return dst;
}

// Rows of a parameter stored as [rows, w]; its element count must be a multiple of w.
long long param_rows(b200_model* m, const std::string& name, long long w) {
    auto it = m->raw.find(name);
    if (it == m->raw.end()) fail(B200_ERR_MISSING_WEIGHT, "missing parameter '%s'", name.c_str());
    if ((long long)it->second.size() % w != 0)
        fail(B200_ERR_INVALID_ARG, "parameter '%s' has %zu elements, not a multiple of %lld", name.c_str(),
             it->second.size(), w);
    return (long long)it->second.size() / w;
}

// Checkpoint names of a transformer layer, each the prefix of its parameters' names up to "weight" / "bias" below the
// layer's own prefix (nullptr: the layer has no such module).  qkv and fc are Linears given as their parts in the
// checkpoint: one fused Linear, or q, k and v, or the gate and x halves; bit j of qkv_bias / fc_bias says part j has a
// bias.
struct LayerNames {
    const char *ln1, *ln2;   // pre-LN: before attention and the MLP; post-LN: after them
    const char* qkv[3];
    const char *out, *attn_ln;
    const char* fc[2];
    const char *mlp_ln, *proj;
    unsigned qkv_bias = 0b111, fc_bias = 0b11;
};
// open_clip ResidualAttentionBlock and timm's ViT Block (SigLIP's vision trunk) have the same arithmetic and the same
// fused q|k|v layout
const LayerNames OPEN_CLIP_BLOCK{"ln_1.", "ln_2.", {"attn.in_proj_"}, "attn.out_proj.", nullptr, {"mlp.c_fc."}, nullptr,
                                 "mlp.c_proj."};
const LayerNames TIMM_BLOCK{"norm1.", "norm2.", {"attn.qkv."}, "attn.proj.", nullptr, {"mlp.fc1."}, nullptr, "mlp.fc2."};
// HF BertLayer and MPNetLayer differ only in their attention half
const LayerNames BERT_LAYER{"attention.output.LayerNorm.", "output.LayerNorm.",
                            {"attention.self.query.", "attention.self.key.", "attention.self.value."},
                            "attention.output.dense.", nullptr, {"intermediate.dense."}, nullptr, "output.dense."};
const LayerNames MPNET_LAYER{"attention.LayerNorm.", "output.LayerNorm.",
                             {"attention.attn.q.", "attention.attn.k.", "attention.attn.v."}, "attention.attn.o.",
                             nullptr, {"intermediate.dense."}, nullptr, "output.dense."};
// NewModel (GTE, verify): up_gate_proj is fused up | gate and has no bias
const LayerNames GTE_LAYER{"attn_ln.", "mlp_ln.", {"attention.qkv_proj."}, "attention.o_proj.", nullptr,
                           {"mlp.up_gate_proj."}, nullptr, "mlp.down_proj.", 0b111, 0b00};
// timm's Eva block (EVA02, verify): k_proj has no bias
const LayerNames EVA_BLOCK{"norm1.", "norm2.", {"attn.q_proj.", "attn.k_proj.", "attn.v_proj."}, "attn.proj.",
                           "attn.norm.", {"mlp.fc1_g.", "mlp.fc1_x."}, "mlp.norm.", "mlp.fc2.", 0b101};

// fp32 parameter `name`, [rows, nb * blk] row-major, with column block i moved to columns i * pblk .. i * pblk + blk - 1
// of [rows, nb * pblk] and zeros in the other columns: replaces the uploaded parameter.
void pad_blocks(b200_model* m, const std::string& name, long long rows, int nb, long long blk, long long pblk) {
    const float* src = param(m, name, rows * nb * blk);
    DeviceBuffer<float> dst((size_t)(rows * nb * pblk));
    MB_CUDA(cudaMemsetAsync(dst.get(), 0, dst.size() * sizeof(float), m->stream));
    for (int i = 0; i < nb; ++i) {
        if (rows == 1)
            MB_CUDA(cudaMemcpyAsync(dst.get() + i * pblk, src + i * blk, blk * sizeof(float), cudaMemcpyDeviceToDevice,
                                    m->stream));
        else
            MB_CUDA(cudaMemcpy2DAsync(dst.get() + i * pblk, nb * pblk * sizeof(float), src + i * blk,
                                      nb * blk * sizeof(float), blk * sizeof(float), rows, cudaMemcpyDeviceToDevice,
                                      m->stream));
    }
    MB_CUDA(cudaStreamSynchronize(m->stream));
    m->raw[name] = std::move(dst);
}

// The zero-padded head layout of a tower whose attention width T.aw exceeds its width (kernel_head_dim): head h of q,
// k and v takes rows h * hdp .. h * hdp + hd - 1 of its part's H * hdp rows of the QKV weight and bias, zero rows and
// zero bias after them, and the out-projection's K dimension has zero columns at the same places.  The QKV GEMM then
// writes exact zeros into the pad columns, QK^T gains exact 0 * 0 terms, the pad columns of the attention output are
// P * 0 = 0 and meet zero weights in the out-projection: the result is the unpadded one up to fp32 summation order.
// Only the CLIP vision towers, whose q|k|v is one fused Linear, have padded heads (check_tower).
void pad_heads(b200_model* m, const TowerW& T, const std::string& p, const LayerNames& nm) {
    const long long w = T.d.width, H = T.d.heads, hd = w / H, hdp = T.aw / H;
    if (hdp == hd) return;
    pad_blocks(m, p + nm.qkv[0] + "weight", 1, (int)(3 * H), hd * w, hdp * w);
    pad_blocks(m, p + nm.qkv[0] + "bias", 1, (int)(3 * H), hd, hdp);
    pad_blocks(m, p + nm.out + "weight", w, (int)H, hd, hdp);
}

// The Linear whose n parts, each [rows, in], are parts[j] under prefix p, as one bf16 weight [n * stride, in] with part
// j at row j * stride and zero rows after each part's own, and its fp32 bias [n * stride] with zeros for a part without
// one (bias_mask), or nullptr when no part has one.  A Linear fused in the checkpoint (one part, no padding) is only
// converted to bf16 and keeps its uploaded bias.  The fp32 weights are released.
void stack_linear(b200_model* m, const std::string& p, const char* const* parts, int n, unsigned bias_mask,
                  long long rows, long long stride, long long in, const __nv_bfloat16*& w_out, const float*& b_out) {
    b_out = nullptr;
    if (n == 1 && rows == stride) {
        w_out = to_bf16(m, p + parts[0] + "weight", rows * in);
        if (bias_mask) b_out = param(m, p + parts[0] + "bias", rows);
        return;
    }
    __nv_bfloat16* w = derived_buffer<__nv_bfloat16>(m, (size_t)(n * stride * in));
    float* b = bias_mask ? derived_buffer<float>(m, (size_t)(n * stride)) : nullptr;
    MB_CUDA(cudaMemsetAsync(w, 0, (size_t)(n * stride * in) * sizeof(__nv_bfloat16), m->stream));
    if (b) MB_CUDA(cudaMemsetAsync(b, 0, (size_t)(n * stride) * sizeof(float), m->stream));
    for (int j = 0; j < n; ++j) {
        const std::string base = p + parts[j];
        kernels::f32_to_bf16(param(m, base + "weight", rows * in), w + (size_t)(j * stride * in), rows * in, m->stream);
        if ((bias_mask >> j) & 1)
            MB_CUDA(cudaMemcpyAsync(b + j * stride, param(m, base + "bias", rows), (size_t)rows * sizeof(float),
                                    cudaMemcpyDeviceToDevice, m->stream));
    }
    MB_CUDA(cudaStreamSynchronize(m->stream));
    for (int j = 0; j < n; ++j) m->raw.erase(p + parts[j] + "weight");
    w_out = w;
    b_out = b;
}

// The columns fc1 writes per token: mlp, or both halves of a gated MLP
int fc1_cols(const TowerW& T) { return T.mlp_form == Mlp::ACT ? T.d.mlp : 2 * T.d.mlp; }

// The layers of T in the layouts run_layers reads.  blocks: the prefix of layer i's names up to the index
// ("visual.transformer.resblocks.", "encoder.layer.", ...).  fc1's parts each have mlp_h rows at a stride of mlp
// (EVA02's gate and x halves, zero rows after each), unless it is one fused Linear of fc1_cols rows; fc2 then gets zero
// K columns at the pad positions, which meet the gated unit's zero pad columns: exact, as for pad_heads.
void build_layers(b200_model* m, TowerW& T, const std::string& blocks, const LayerNames& nm) {
    const long long w = T.d.width, aw = T.aw, mlp = T.d.mlp, fc = fc1_cols(T);
    const int n_qkv = nm.qkv[1] ? 3 : 1, n_fc = nm.fc[1] ? 2 : 1;
    const long long fc_rows = n_fc == 1 ? fc : T.mlp_h;
    auto norm = [&](const std::string& p, const char* name, long long n, const float*& g, const float*& b) {
        g = param(m, p + name + "weight", n);
        b = param(m, p + name + "bias", n);
    };
    T.layers.resize(T.d.layers);
    for (int i = 0; i < T.d.layers; ++i) {
        const std::string p = blocks + std::to_string(i) + ".";
        LayerW& L = T.layers[i];
        norm(p, nm.ln1, w, L.ln1_w, L.ln1_b);
        pad_heads(m, T, p, nm);
        stack_linear(m, p, nm.qkv, n_qkv, nm.qkv_bias, 3 * aw / n_qkv, 3 * aw / n_qkv, w, L.w_qkv, L.b_qkv);
        L.w_o = to_bf16(m, p + nm.out + "weight", w * aw);
        L.b_o = param(m, p + nm.out + "bias", w);
        if (nm.attn_ln) norm(p, nm.attn_ln, w, L.ln_attn_w, L.ln_attn_b);
        if (n_fc == 1 && fc != mlp) {   // a fused gated fc1 (GTE's up | gate) holds both halves
            const std::string fw = p + nm.fc[0] + "weight";
            const long long rows = param_rows(m, fw, w);
            MB_CHECK_ARG(rows == fc, "%s has %lld rows, 2 * mlp = %lld are needed", fw.c_str(), rows, fc);
        }
        stack_linear(m, p, nm.fc, n_fc, nm.fc_bias, fc_rows, fc / n_fc, w, L.w_fc, L.b_fc);
        if (nm.mlp_ln) norm(p, nm.mlp_ln, T.mlp_h, L.ln_mlp_w, L.ln_mlp_b);
        if (T.mlp_h != mlp) pad_blocks(m, p + nm.proj + "weight", w, 1, T.mlp_h, mlp);
        L.w_proj = to_bf16(m, p + nm.proj + "weight", w * mlp);
        L.b_proj = param(m, p + nm.proj + "bias", w);
        norm(p, nm.ln2, w, L.ln2_w, L.ln2_b);
    }
}

// transformers MPNetEncoder.relative_position_bucket for relative_position = key - query, in the same fp32 arithmetic:
// n = query - key; keys after the query take the upper half of the buckets; |n| < half / 2 is exact, larger distances
// are log-spaced up to max_distance, truncated toward zero.
int relative_position_bucket(int rel, int num_buckets, int max_distance) {
    const int half = num_buckets / 2, max_exact = half / 2;
    const int base = rel > 0 ? half : 0;
    const int n = rel < 0 ? -rel : rel;
    if (n < max_exact) return base + n;
    const float lg = std::log((float)n / (float)max_exact) / (float)std::log((double)max_distance / max_exact);
    const int large = max_exact + (int)(lg * (float)(half - max_exact));
    return base + std::min(large, half - 1);
}

// MPNet's relative-position bias, built once per handle: table[h][d + ctx - 1] = weight[bucket(d)][h] * log2(e) for
// every key - query distance d of a sequence of up to ctx tokens.  Every layer reads the same table (a fixed pointer,
// so captured CUDA graphs replay it).
attention::RelBias build_rel_bias(b200_model* m, const TowerW& T) {
    const int H = T.d.heads, nb = m->desc.rel_buckets, smax = T.d.ctx, span = 2 * smax - 1;
    const float* w = param(m, "encoder.relative_attention_bias.weight", (long long)nb * H);
    std::vector<float> wh((size_t)nb * H), table((size_t)H * span);
    MB_CUDA(cudaMemcpy(wh.data(), w, wh.size() * sizeof(float), cudaMemcpyDeviceToHost));
    for (int d = -(smax - 1); d <= smax - 1; ++d) {
        const int bucket = relative_position_bucket(d, nb, m->desc.rel_max_distance);
        for (int h = 0; h < H; ++h) table[(size_t)h * span + d + smax - 1] = wh[(size_t)bucket * H + h] * 1.4426950408889634f;
    }
    float* dev = derived_buffer<float>(m, table.size());
    MB_CUDA(cudaMemcpy(dev, table.data(), table.size() * sizeof(float), cudaMemcpyHostToDevice));
    attention::RelBias b;
    b.table = dev;
    b.smax = smax;
    return b;
}

std::vector<float> to_host(const float* d, size_t n) {
    std::vector<float> h(n);
    MB_CUDA(cudaMemcpy(h.data(), d, n * sizeof(float), cudaMemcpyDeviceToHost));
    return h;
}

const float* upload_derived(b200_model* m, const std::vector<float>& h) {
    float* d = derived_buffer<float>(m, h.size());
    MB_CUDA(cudaMemcpy(d, h.data(), h.size() * sizeof(float), cudaMemcpyHostToDevice));
    return d;
}

// A timm trunk's pos_embed with the patch conv's bias folded into its patch rows: the bias is the same for every patch,
// so pos[t] + bias + conv(patch) == pos'[t] + conv(patch); the class rows have no conv term.
const float* fold_patch_bias(b200_model* m, const TowerW& T, const std::string& trunk) {
    const long long w = T.d.width;
    std::vector<float> pos = to_host(param(m, trunk + "pos_embed", (long long)T.tokens * w), (size_t)T.tokens * w);
    const std::vector<float> bias = to_host(param(m, trunk + "patch_embed.proj.bias", w), (size_t)w);
    for (long long i = T.cls_rows * w; i < (long long)pos.size(); ++i) pos[i] += bias[i % w];
    return upload_derived(m, pos);
}

// SigLIP's timm trunk after the patch conv (open_clip names, verify): pos_embed with the conv bias folded in, the
// blocks, the final norm and the MAP head, whose latent query projection q = latent W_q^T + b_q is computed here once,
// in double.
void build_siglip_vision(b200_model* m, TowerW& T) {
    const long long w = T.d.width;
    const std::string t = "visual.trunk.";
    T.pos = fold_patch_bias(m, T, t);
    build_layers(m, T, t + "blocks.", TIMM_BLOCK);
    T.ln_out_w = param(m, t + "norm.weight", w);
    T.ln_out_b = param(m, t + "norm.bias", w);
    const std::string a = t + "attn_pool.";
    const std::vector<float> latent = to_host(param(m, a + "latent", w), (size_t)w);
    const std::vector<float> wq = to_host(param(m, a + "q.weight", w * w), (size_t)(w * w));
    const std::vector<float> bq = to_host(param(m, a + "q.bias", w), (size_t)w);
    std::vector<float> q((size_t)w);
    for (long long o = 0; o < w; ++o) {
        double acc = bq[o];
        for (long long i = 0; i < w; ++i) acc += (double)wq[o * w + i] * latent[i];
        q[o] = (float)acc;
    }
    MapW& P = T.map;
    P.q = upload_derived(m, q);
    P.w_kv = to_bf16(m, a + "kv.weight", 2 * w * w);
    P.b_kv = param(m, a + "kv.bias", 2 * w);
    P.w_proj = to_bf16(m, a + "proj.weight", w * w);
    P.b_proj = param(m, a + "proj.bias", w);
    P.ln_w = param(m, a + "norm.weight", w);
    P.ln_b = param(m, a + "norm.bias", w);
    const long long mlp = param_rows(m, a + "mlp.fc1.weight", w);
    MB_CHECK_ARG(mlp > 0 && mlp % 64 == 0, "%smlp.fc1 has %lld rows: a positive multiple of 64 is needed", a.c_str(), mlp);
    P.mlp = (int)mlp;
    P.w_fc1 = to_bf16(m, a + "mlp.fc1.weight", mlp * w);
    P.b_fc1 = param(m, a + "mlp.fc1.bias", mlp);
    P.w_fc2 = to_bf16(m, a + "mlp.fc2.weight", w * mlp);
    P.b_fc2 = param(m, a + "mlp.fc2.bias", w);
}

// conv + BatchNorm of the ResNet tower -> ConvW (see ConvW)
ConvW fold_conv_bn(b200_model* m, const std::string& conv, const std::string& bn, int cin, int cout, int k) {
    const long long nw = (long long)cout * cin * k * k;
    const std::vector<float> w = to_host(param(m, conv + ".weight", nw), (size_t)nw);
    const std::vector<float> g = to_host(param(m, bn + ".weight", cout), (size_t)cout);
    const std::vector<float> beta = to_host(param(m, bn + ".bias", cout), (size_t)cout);
    const std::vector<float> mean = to_host(param(m, bn + ".running_mean", cout), (size_t)cout);
    const std::vector<float> var = to_host(param(m, bn + ".running_var", cout), (size_t)cout);
    std::vector<double> scale((size_t)cout);
    std::vector<float> bias((size_t)cout);
    for (int o = 0; o < cout; ++o) {
        scale[o] = (double)g[o] / std::sqrt((double)var[o] + 1e-5);
        bias[o] = (float)((double)beta[o] - (double)mean[o] * scale[o]);
    }
    const int K = gemm::conv_rows_k(cin, k);
    std::vector<float> rows((size_t)cout * K);
    gemm::conv_weight_rows(w.data(), cout, cin, k, scale.data(), rows.data());
    // Both copies go on the model's stream: a cudaMemcpy from pageable memory may return before its DMA lands, and the
    // conversion below runs on the (non-blocking) model stream, which would not wait for it.
    DeviceBuffer<float> tmp(rows.size());
    MB_CUDA(cudaMemcpyAsync(tmp.get(), rows.data(), rows.size() * sizeof(float), cudaMemcpyHostToDevice, m->stream));
    __nv_bfloat16* wb = derived_buffer<__nv_bfloat16>(m, rows.size());
    kernels::f32_to_bf16(tmp.get(), wb, (long long)rows.size(), m->stream);
    float* db = derived_buffer<float>(m, bias.size());
    MB_CUDA(cudaMemcpyAsync(db, bias.data(), bias.size() * sizeof(float), cudaMemcpyHostToDevice, m->stream));
    MB_CUDA(cudaStreamSynchronize(m->stream));
    m->raw.erase(conv + ".weight");
    ConvW c;
    c.w = wb;
    c.b = db;
    c.cin = cin;
    c.cout = cout;
    c.k = k;
    return c;
}

// The ResNet tower's folded weights, the attention pool and the activation buffers (ResnetW).
void build_resnet(b200_model* m, TowerW& T) {
    ResnetW& R = m->resnet;
    const b200_model_desc& d = m->desc;
    const int width = d.resnet_width, S = d.resnet_image_size, E = d.embed_dim;
    const std::string v = "visual.";
    R.stem[0] = fold_conv_bn(m, v + "conv1", v + "bn1", 3, width / 2, 3);
    R.stem[1] = fold_conv_bn(m, v + "conv2", v + "bn2", width / 2, width / 2, 3);
    R.stem[2] = fold_conv_bn(m, v + "conv3", v + "bn3", width / 2, width, 3);
    // per_image: the largest activation of one image (stem im2col rows are 64 wide)
    long long H = S / 4, per_image = (long long)(S / 2) * (S / 2) * std::max(64, width);
    int inplanes = width;
    for (int s = 0; s < 4; ++s) {
        const int planes = width << s;
        for (int i = 0; i < d.resnet_layers[s]; ++i) {
            const std::string p = v + "layer" + std::to_string(s + 1) + "." + std::to_string(i) + ".";
            BottleneckW B;
            B.stride = i == 0 && s > 0 ? 2 : 1;
            B.c1 = fold_conv_bn(m, p + "conv1", p + "bn1", inplanes, planes, 1);
            B.c2 = fold_conv_bn(m, p + "conv2", p + "bn2", planes, planes, 3);
            B.c3 = fold_conv_bn(m, p + "conv3", p + "bn3", planes, 4 * planes, 1);
            B.has_ds = B.stride > 1 || inplanes != 4 * planes;
            if (B.has_ds) B.ds = fold_conv_bn(m, p + "downsample.0", p + "downsample.1", inplanes, 4 * planes, 1);
            per_image = std::max({per_image, H * H * inplanes, H * H * planes});
            H /= B.stride;
            per_image = std::max(per_image, H * H * 4 * planes);
            inplanes = 4 * planes;
            R.blocks.push_back(B);
        }
    }
    R.C = inplanes;
    R.grid = (int)H;
    const long long C = R.C, tokens = H * H + 1;
    T.grid = (int)H;
    T.tokens = (int)tokens;
    per_image = std::max(per_image, tokens * 2 * C);   // the K|V rows (the tokens and the fp32 query are smaller)
    const std::string a = v + "attnpool.";
    R.pos = param(m, a + "positional_embedding", tokens * C);
    __nv_bfloat16* wkv = derived_buffer<__nv_bfloat16>(m, (size_t)(2 * C * C));
    float* bkv = derived_buffer<float>(m, (size_t)(2 * C));
    const char* kv_names[2] = {"k_proj", "v_proj"};
    for (int j = 0; j < 2; ++j) {
        kernels::f32_to_bf16(param(m, a + kv_names[j] + ".weight", C * C), wkv + (size_t)j * C * C, C * C, m->stream);
        MB_CUDA(cudaMemcpyAsync(bkv + (size_t)j * C, param(m, a + kv_names[j] + ".bias", C), (size_t)C * 4,
                                cudaMemcpyDeviceToDevice, m->stream));
    }
    MB_CUDA(cudaStreamSynchronize(m->stream));
    for (int j = 0; j < 2; ++j) m->raw.erase(a + kv_names[j] + ".weight");
    R.w_kv = wkv;
    R.b_kv = bkv;
    R.w_q = to_bf16(m, a + "q_proj.weight", C * C);
    R.b_q = param(m, a + "q_proj.bias", C);
    R.w_c = to_bf16(m, a + "c_proj.weight", (long long)E * C);
    R.b_c = param(m, a + "c_proj.bias", E);
    for (auto& b : R.buf) b = DeviceBuffer<__nv_bfloat16>((size_t)d.max_batch * per_image);
}

// host fp32 values -> an owned bf16 device copy.  The copy goes on the model's stream ahead of the conversion: a
// cudaMemcpy from pageable memory may return before its DMA lands, and the non-blocking model stream would not wait.
const __nv_bfloat16* upload_bf16(b200_model* m, const std::vector<float>& h) {
    DeviceBuffer<float> tmp(h.size());
    MB_CUDA(cudaMemcpyAsync(tmp.get(), h.data(), h.size() * sizeof(float), cudaMemcpyHostToDevice, m->stream));
    __nv_bfloat16* dst = derived_buffer<__nv_bfloat16>(m, h.size());
    kernels::f32_to_bf16(tmp.get(), dst, (long long)h.size(), m->stream);
    MB_CUDA(cudaStreamSynchronize(m->stream));
    return dst;
}

// the MLP activation of open_clip's towers
int open_clip_act(const b200_model_desc& d) {
    return d.act == B200_ACT_QUICKGELU ? gemm::ACT_QUICKGELU : gemm::ACT_GELU;
}

// open_clip's VisionTransformer or SigLIP's timm trunk: the patch conv (conv_name, no bias) in both GEMM layouts, then
// the rest of the tower.
void build_vit(b200_model* m, TowerW& T, const char* conv_name, int cls_rows) {
    const long long w = T.d.width, p = T.d.patch;
    T.grid = T.d.image_size / T.d.patch;
    T.cls_rows = cls_rows;
    T.tokens = T.grid * T.grid + T.cls_rows;
    const int K = 3 * (int)p * (int)p;
    T.kpad = (int)round_up((size_t)K, 64);
    const float* conv = param(m, conv_name, w * K);
    __nv_bfloat16* cw = derived_buffer<__nv_bfloat16>(m, (size_t)w * T.kpad);
    kernels::pad_rows_to_bf16(conv, (int)w, K, T.kpad, cw, m->stream);
    MB_CUDA(cudaStreamSynchronize(m->stream));
    T.conv_w = cw;
    __nv_bfloat16* cg = derived_buffer<__nv_bfloat16>(m, (size_t)w * gemm::patch_gather_k((int)p));
    kernels::patch_weight_rows(conv, (int)w, (int)p, gemm::patch_gather_kbpd((int)p), cg, m->stream);
    MB_CUDA(cudaStreamSynchronize(m->stream));
    T.conv_wg = cg;
}

// The EVA02 trunk (open_clip TimmModel over timm's Eva, verify): pos_embed with the patch conv's bias folded in, the
// RoPE table of the grid (built in fp64 on the host), the blocks (EVA_BLOCK: q | k | v with a zero k bias, fc1_g | fc1_x
// with the hidden size padded to a multiple of 64), the final norm and the head Linear [E, w] with its bias.
void build_eva_vision(b200_model* m, TowerW& T) {
    const std::string t = "visual.trunk.";
    build_vit(m, T, "visual.trunk.patch_embed.proj.weight", 1);
    const long long w = T.d.width, E = m->desc.embed_dim;
    T.eps = m->desc.layer_norm_eps;
    T.cls = param(m, t + "cls_token", w);
    T.pos = fold_patch_bias(m, T, t);
    std::vector<float> rope((size_t)T.grid * T.grid * 64);
    kernels::rope_table(T.grid, m->desc.eva_rope_ref_grid, rope.data());
    T.rope = upload_derived(m, rope);
    T.rope_first = 1;
    T.mlp_form = Mlp::SWIGLU_LN;
    // the SwiGLU hidden size is the checkpoint's; it must be the one the model was created with
    const long long h = param_rows(m, t + "blocks.0.mlp.fc1_g.weight", w);
    MB_CHECK_ARG(h == T.d.mlp, "EVA02: %sblocks.0.mlp.fc1_g has %lld rows, vision.mlp is %d", t.c_str(), h, T.d.mlp);
    T.d.mlp = (int)round_up((size_t)h, 64);
    build_layers(m, T, t + "blocks.", EVA_BLOCK);
    T.ln_out_w = param(m, t + "norm.weight", w);
    T.ln_out_b = param(m, t + "norm.bias", w);
    T.w_tproj = to_bf16(m, t + "head.weight", E * w);
    T.b_tproj = param(m, t + "head.bias", E);
}

// The ConvNeXt tower's weights in the layouts its kernels read (ConvnextW) and its activation buffers.  T holds the
// stem as a patch-4 ViT patch embedding.
void build_convnext(b200_model* m, TowerW& T) {
    ConvnextW& X = m->convnext;
    const b200_model_desc& d = m->desc;
    const long long E = d.embed_dim;
    const std::string t = "visual.trunk.";
    build_vit(m, T, "visual.trunk.stem.0.weight", 0);
    X.stem_b = param(m, t + "stem.0.bias", T.d.width);
    X.stem_ln_w = param(m, t + "stem.1.weight", T.d.width);
    X.stem_ln_b = param(m, t + "stem.1.bias", T.d.width);
    long long prev = 0;
    for (int s = 0; s < 4; ++s) {
        ConvnextStageW& st = X.stages[s];
        const long long C = d.convnext_dims[s];
        st.C = (int)C;
        const std::string p = t + "stages." + std::to_string(s) + ".";
        if (s > 0) {
            st.ds_ln_w = param(m, p + "downsample.0.weight", prev);
            st.ds_ln_b = param(m, p + "downsample.0.bias", prev);
            // [C, C_prev, 2, 2] -> [C, (dy * 2 + dx) * C_prev + c]: ln_pixels' patch row order
            const std::vector<float> w = to_host(param(m, p + "downsample.1.weight", C * prev * 4), (size_t)(C * prev * 4));
            std::vector<float> rows(w.size());
            for (long long o = 0; o < C; ++o)
                for (long long c = 0; c < prev; ++c)
                    for (int q = 0; q < 4; ++q) rows[(o * 4 + q) * prev + c] = w[(o * prev + c) * 4 + q];
            st.ds_w = upload_bf16(m, rows);
            m->raw.erase(p + "downsample.1.weight");
            st.ds_b = param(m, p + "downsample.1.bias", C);
        }
        st.blocks.resize(d.convnext_depths[s]);
        for (int i = 0; i < d.convnext_depths[s]; ++i) {
            const std::string b = p + "blocks." + std::to_string(i) + ".";
            ConvnextBlockW& B = st.blocks[i];
            // conv_dw.weight [C, 1, 7, 7] -> [49, C]: a tap's channels contiguous
            const std::vector<float> dw = to_host(param(m, b + "conv_dw.weight", C * 49), (size_t)(C * 49));
            std::vector<float> taps(dw.size());
            for (long long c = 0; c < C; ++c)
                for (int k = 0; k < 49; ++k) taps[k * C + c] = dw[c * 49 + k];
            B.dw_w = upload_derived(m, taps);
            m->raw.erase(b + "conv_dw.weight");
            B.dw_b = param(m, b + "conv_dw.bias", C);
            B.ln_w = param(m, b + "norm.weight", C);
            B.ln_b = param(m, b + "norm.bias", C);
            B.w1 = to_bf16(m, b + "mlp.fc1.weight", 4 * C * C);
            B.b1 = param(m, b + "mlp.fc1.bias", 4 * C);
            // gamma * (u W2^T + b2) == u (gamma W2)^T + gamma b2
            const std::vector<float> g = to_host(param(m, b + "gamma", C), (size_t)C);
            std::vector<float> w2 = to_host(param(m, b + "mlp.fc2.weight", 4 * C * C), (size_t)(4 * C * C));
            std::vector<float> b2 = to_host(param(m, b + "mlp.fc2.bias", C), (size_t)C);
            for (long long o = 0; o < C; ++o) {
                for (long long k = 0; k < 4 * C; ++k) w2[o * 4 * C + k] *= g[o];
                b2[o] *= g[o];
            }
            B.w2 = upload_bf16(m, w2);
            B.b2 = upload_derived(m, b2);
            for (const char* nm : {"mlp.fc2.weight", "mlp.fc2.bias", "gamma"}) m->raw.erase(b + nm);
        }
        prev = C;
    }
    X.head_ln_w = param(m, t + "head.norm.weight", prev);
    X.head_ln_b = param(m, t + "head.norm.bias", prev);
    if (d.convnext_head == 0) {
        X.w_proj = to_bf16(m, "visual.head.proj.weight", E * prev);
    } else {
        X.w_fc1 = to_bf16(m, "visual.head.mlp.fc1.weight", 2 * E * prev);
        X.b_fc1 = param(m, "visual.head.mlp.fc1.bias", 2 * E);
        X.w_fc2 = to_bf16(m, "visual.head.mlp.fc2.weight", E * 2 * E);
    }
    // x fp32, h bf16, u bf16 (4 C wide) of the first stage, capped at ~24 GB like the transformer workspaces; the
    // head's rows (n x C3, n x 2E) fit in h and u
    const long long per_image = (long long)T.tokens * T.d.width;
    X.max_images = (int)std::max<long long>(1, std::min<long long>(d.max_batch, (24LL << 30) / (per_image * 14)));
    X.x = DeviceBuffer<float>((size_t)X.max_images * per_image);
    X.h = DeviceBuffer<__nv_bfloat16>((size_t)X.max_images * per_image);
    X.u = DeviceBuffer<__nv_bfloat16>((size_t)X.max_images * per_image * 4);
}

// CoCa's attentional pooler (open_clip AttentionalPooler, verify) after the CLIP ViT trunk: ln_k over the trunk's
// width, the K and V projections stacked into one Linear [2d, width] with in_proj_bias[d:3d], out_proj, and q0 =
// ln_q(query[0]) W_q^T + b_q, computed here once in double; then ln_post and proj over d = embed_dim.
constexpr long long COCA_POOL_QUERIES = 256;   // open_clip CoCa's attn_pooler_queries: the rows of attn_pool.query

void build_coca_pooler(b200_model* m, TowerW& T) {
    const long long w = T.d.width, d = m->desc.embed_dim;
    const std::string a = "visual.attn_pool.";
    MapW& P = T.map;
    // only query 0 is read: the queries do not interact and the embedding pools query 0
    const std::vector<float> query = to_host(param(m, a + "query", COCA_POOL_QUERIES * d), (size_t)d);
    const std::vector<float> gq = to_host(param(m, a + "ln_q.weight", d), (size_t)d);
    const std::vector<float> bln = to_host(param(m, a + "ln_q.bias", d), (size_t)d);
    const std::vector<float> wq = to_host(param(m, a + "attn.q_proj_weight", d * d), (size_t)(d * d));
    const float* in_bias = param(m, a + "attn.in_proj_bias", 3 * d);
    const std::vector<float> bq = to_host(in_bias, (size_t)d);
    double mean = 0, var = 0;
    for (long long i = 0; i < d; ++i) mean += query[i];
    mean /= (double)d;
    for (long long i = 0; i < d; ++i) var += ((double)query[i] - mean) * ((double)query[i] - mean);
    const double rstd = 1.0 / std::sqrt(var / (double)d + 1e-5);
    std::vector<double> lq((size_t)d);
    for (long long i = 0; i < d; ++i) lq[i] = ((double)query[i] - mean) * rstd * gq[i] + bln[i];
    std::vector<float> q((size_t)d);
    for (long long o = 0; o < d; ++o) {
        double acc = bq[o];
        for (long long i = 0; i < d; ++i) acc += (double)wq[o * d + i] * lq[i];
        q[o] = (float)acc;
    }
    P.q = upload_derived(m, q);
    for (const char* nm : {"query", "ln_q.weight", "ln_q.bias", "attn.q_proj_weight"}) m->raw.erase(a + nm);
    P.ln_w = param(m, a + "ln_k.weight", w);
    P.ln_b = param(m, a + "ln_k.bias", w);
    static const char* const kv_parts[2] = {"attn.k_proj_", "attn.v_proj_"};
    stack_linear(m, a, kv_parts, 2, 0, d, d, w, P.w_kv, P.b_kv);
    P.b_kv = in_bias + d;
    P.w_proj = to_bf16(m, a + "attn.out_proj.weight", d * d);
    P.b_proj = param(m, a + "attn.out_proj.bias", d);
    T.ln_out_w = param(m, "visual.ln_post.weight", d);
    T.ln_out_b = param(m, "visual.ln_post.bias", d);
    T.proj = param(m, "visual.proj", d * m->desc.embed_dim);
}

// OWL-ViT's detection head (OwlW) under the checkpoint's own names, and its box bias table, built in fp64 on the host.
void build_owl(b200_model* m, const TowerW& T) {
    OwlW& D = m->owl;
    const long long w = T.d.width, E = m->desc.embed_dim;
    D.ln_w = param(m, "layer_norm.weight", w);
    D.ln_b = param(m, "layer_norm.bias", w);
    D.ncls = (int)round_up((size_t)E + 2, 64);
    std::vector<float> rows((size_t)D.ncls * w, 0.f), bias((size_t)D.ncls, 0.f);
    const struct {
        const char* name;
        long long n;
    } parts[3] = {{"class_head.dense0.", E}, {"class_head.logit_shift.", 1}, {"class_head.logit_scale.", 1}};
    long long at = 0;
    for (const auto& pt : parts) {
        const std::string p = pt.name;
        const std::vector<float> wt = to_host(param(m, p + "weight", pt.n * w), (size_t)(pt.n * w));
        const std::vector<float> bt = to_host(param(m, p + "bias", pt.n), (size_t)pt.n);
        std::copy(wt.begin(), wt.end(), rows.begin() + at * w);
        std::copy(bt.begin(), bt.end(), bias.begin() + at);
        m->raw.erase(p + "weight");
        m->raw.erase(p + "bias");
        at += pt.n;
    }
    D.w_cls = upload_bf16(m, rows);
    D.b_cls = upload_derived(m, bias);
    D.w_box0 = to_bf16(m, "box_head.dense0.weight", w * w);
    D.b_box0 = param(m, "box_head.dense0.bias", w);
    D.w_box1 = to_bf16(m, "box_head.dense1.weight", w * w);
    D.b_box1 = param(m, "box_head.dense1.bias", w);
    D.w_box2 = param(m, "box_head.dense2.weight", 4 * w);
    D.b_box2 = param(m, "box_head.dense2.bias", 4);
    std::vector<float> bb((size_t)T.grid * T.grid * 4);
    kernels::owl_box_bias(T.grid, bb.data());
    D.box_bias = upload_derived(m, bb);
}

// LanguageBind's video tower (languagebind/video/modeling_video.py:698-785, verify) under the CLIP ViT names, its frames
// laid out (b T + t) N + token.  visual.class_embedding is [width] (CLIPVisionEmbeddings) or one row per frame [T,
// width] (CLIPVisionEmbeddings3D with tube 1); it and visual.positional_embedding become one table of a video's T N rows
// (frame t's class row: class_embedding[t] + positional_embedding[0], its patch rows: positional_embedding), which
// vit_embed_rows writes and the patch GEMM adds conv1 onto.  Per layer the temporal step's weights (LayerW), and the
// head: ln_post, visual.proj [width, E] and exp(logit_scale).
void build_video_vision(b200_model* m, TowerW& T) {
    const long long w = T.d.width, F = m->desc.video_frames;
    build_vit(m, T, "visual.conv1.weight", 1);
    T.act = open_clip_act(m->desc);
    T.frames = (int)F;
    const long long N = T.tokens;
    const long long cls_rows = param_rows(m, "visual.class_embedding", w);
    MB_CHECK_ARG(cls_rows == 1 || cls_rows == F, "visual.class_embedding has %lld rows: 1 or video_frames (%lld)",
                 cls_rows, F);
    const std::vector<float> cls = to_host(param(m, "visual.class_embedding", cls_rows * w), (size_t)(cls_rows * w));
    const std::vector<float> pos = to_host(param(m, "visual.positional_embedding", N * w), (size_t)(N * w));
    std::vector<float> table((size_t)(F * N * w));
    for (long long t = 0; t < F; ++t) {
        std::copy(pos.begin(), pos.end(), table.begin() + t * N * w);
        const float* c = cls.data() + (cls_rows == 1 ? 0 : t * w);
        for (long long i = 0; i < w; ++i) table[(size_t)(t * N * w + i)] = c[i] + pos[(size_t)i];
    }
    T.pos = upload_derived(m, table);
    m->raw.erase("visual.class_embedding");
    m->raw.erase("visual.positional_embedding");
    T.ln_pre_w = param(m, "visual.ln_pre.weight", w);
    T.ln_pre_b = param(m, "visual.ln_pre.bias", w);
    build_layers(m, T, "visual.transformer.resblocks.", OPEN_CLIP_BLOCK);
    static const char* const tqkv[1] = {"temporal_attn.in_proj_"};
    for (int i = 0; i < T.d.layers; ++i) {
        const std::string p = "visual.transformer.resblocks." + std::to_string(i) + ".";
        LayerW& L = T.layers[i];
        const float* temb = param(m, p + "temporal_embedding", F * w);
        L.temb = F > 1 ? temb : nullptr;   // one frame adds none (modeling_video.py:214)
        L.tln_w = param(m, p + "temporal_ln_1.weight", w);
        L.tln_b = param(m, p + "temporal_ln_1.bias", w);
        stack_linear(m, p, tqkv, 1, 0b1, 3 * w, 3 * w, w, L.w_tqkv, L.b_tqkv);
        L.w_to = to_bf16(m, p + "temporal_attn.out_proj.weight", w * w);
        L.b_to = param(m, p + "temporal_attn.out_proj.bias", w);
    }
    T.ln_out_w = param(m, "visual.ln_post.weight", w);
    T.ln_out_b = param(m, "visual.ln_post.bias", w);
    T.proj = param(m, "visual.proj", w * m->desc.embed_dim);
    T.out_scale = std::exp(to_host(param(m, "logit_scale", 1), 1)[0]);
}

void build_vision(b200_model* m) {
    TowerW& T = m->vision;
    const long long w = T.d.width;
    switch (m->kind.vision) {
    case VisionKind::CLIP_VIT:
    case VisionKind::COCA_VIT:
        build_vit(m, T, "visual.conv1.weight", 1);
        T.act = open_clip_act(m->desc);
        T.cls = param(m, "visual.class_embedding", w);
        T.pos = param(m, "visual.positional_embedding", (long long)T.tokens * w);
        T.ln_pre_w = param(m, "visual.ln_pre.weight", w);
        T.ln_pre_b = param(m, "visual.ln_pre.bias", w);
        build_layers(m, T, "visual.transformer.resblocks.", OPEN_CLIP_BLOCK);
        if (m->kind.vision == VisionKind::COCA_VIT) {
            build_coca_pooler(m, T);
            break;
        }
        T.ln_out_w = param(m, "visual.ln_post.weight", w);
        T.ln_out_b = param(m, "visual.ln_post.bias", w);
        if (m->desc.owl_detect)
            build_owl(m, T);
        else
            T.proj = param(m, "visual.proj", w * m->desc.embed_dim);
        break;
    case VisionKind::SIGLIP_VIT:
        build_vit(m, T, "visual.trunk.patch_embed.proj.weight", 0);
        T.act = open_clip_act(m->desc);
        T.eps = m->desc.layer_norm_eps;
        build_siglip_vision(m, T);
        break;
    case VisionKind::RESNET:
        build_resnet(m, T);
        break;
    case VisionKind::CONVNEXT:
        build_convnext(m, T);
        break;
    case VisionKind::EVA_VIT:
        build_eva_vision(m, T);
        break;
    case VisionKind::VIDEO_VIT:
        build_video_vision(m, T);
        break;
    }
}

void build_text(b200_model* m) {
    TowerW& T = m->text;
    const long long w = T.d.width, E = m->desc.embed_dim;
    if (m->kind.text != TextKind::NONE) T.tokens = T.d.ctx;
    switch (m->kind.text) {
    case TextKind::CLIP:
    case TextKind::COCA:
    case TextKind::SIGLIP: {
        const bool siglip = m->kind.text == TextKind::SIGLIP;
        // SigLIP, EVA02 (open_clip CustomTextCLIP) and CoCa keep the text tower under "text."
        const std::string p =
            siglip || m->desc.arch == B200_ARCH_CLIP_EVA || m->kind.text == TextKind::COCA ? "text." : "";
        if (m->kind.text == TextKind::COCA) T.text_cls = param(m, p + "cls_emb", w);
        T.act = open_clip_act(m->desc);
        T.tok = param(m, p + "token_embedding.weight", (long long)T.d.vocab * w);
        T.pos = param(m, p + "positional_embedding", (long long)T.d.ctx * w);
        build_layers(m, T, p + "transformer.resblocks.", OPEN_CLIP_BLOCK);
        T.ln_out_w = param(m, p + "ln_final.weight", w);
        T.ln_out_b = param(m, p + "ln_final.bias", w);
        if (siglip) {
            T.eps = m->desc.layer_norm_eps;
            T.w_tproj = to_bf16(m, "text.text_projection.weight", E * w);
            T.b_tproj = param(m, "text.text_projection.bias", E);
        } else {
            T.proj = param(m, p + "text_projection", w * E);
        }
        break;
    }
    case TextKind::BERT: {
        T.eps = 1e-12f;   // BertConfig's layer_norm_eps
        T.pre_ln = false;
        T.tok = param(m, "embeddings.word_embeddings.weight", (long long)T.d.vocab * w);
        T.pos = param(m, "embeddings.position_embeddings.weight", (long long)T.d.ctx * w);
        const int tv = std::max(1, m->desc.type_vocab);
        T.type0 = param(m, "embeddings.token_type_embeddings.weight", (long long)tv * w);  // row 0 is used
        T.emb_ln_w = param(m, "embeddings.LayerNorm.weight", w);
        T.emb_ln_b = param(m, "embeddings.LayerNorm.bias", w);
        build_layers(m, T, "encoder.layer.", BERT_LAYER);
        if (m->desc.cls_labels > 0) {
            T.pool_w = param(m, "pooler.dense.weight", w * w);
            T.pool_b = param(m, "pooler.dense.bias", w);
            T.cls_w = param(m, "classifier.weight", E * w);   // E == cls_labels
            T.cls_b = param(m, "classifier.bias", E);
        }
        break;
    }
    case TextKind::ROBERTA: {
        T.eps = m->desc.layer_norm_eps;
        T.pre_ln = false;
        T.tok = param(m, "embeddings.word_embeddings.weight", (long long)T.d.vocab * w);
        // positions run pad_id + 1 .. pad_id + ctx (pads take pad_id): the table has at least ctx + pad_id + 1 rows
        const long long pos_rows = param_rows(m, "embeddings.position_embeddings.weight", w);
        MB_CHECK_ARG(pos_rows >= (long long)T.d.ctx + m->desc.pad_id + 1,
                     "embeddings.position_embeddings has %lld rows; %d tokens with pad id %d need %d", pos_rows,
                     T.d.ctx, m->desc.pad_id, T.d.ctx + m->desc.pad_id + 1);
        T.pos = param(m, "embeddings.position_embeddings.weight", pos_rows * w);
        T.emb_ln_w = param(m, "embeddings.LayerNorm.weight", w);
        T.emb_ln_b = param(m, "embeddings.LayerNorm.bias", w);
        if (m->kind.mpnet) {
            build_layers(m, T, "encoder.layer.", MPNET_LAYER);
            T.rel_bias = build_rel_bias(m, T);
        } else {
            T.type0 = param(m, "embeddings.token_type_embeddings.weight", w);   // type_vocab_size 1
            build_layers(m, T, "encoder.layer.", BERT_LAYER);
        }
        break;
    }
    case TextKind::GTE: {
        T.eps = m->desc.layer_norm_eps;
        T.pre_ln = false;
        T.mlp_form = Mlp::GEGLU;
        T.tok = param(m, "embeddings.word_embeddings.weight", (long long)T.d.vocab * w);
        const int tv = std::max(1, m->desc.type_vocab);
        T.type0 = param(m, "embeddings.token_type_embeddings.weight", (long long)tv * w);  // row 0 is used
        T.emb_ln_w = param(m, "embeddings.LayerNorm.weight", w);
        T.emb_ln_b = param(m, "embeddings.LayerNorm.bias", w);
        build_layers(m, T, "encoder.layer.", GTE_LAYER);
        std::vector<float> rope((size_t)T.d.ctx * 64);
        kernels::rope_table_ntk(T.d.ctx, m->desc.rope_theta, m->desc.rope_ntk_factor, rope.data());
        T.rope = upload_derived(m, rope);
        T.rope_pairing = kernels::RopePairing::HALF;
        break;
    }
    }
    if (m->desc.text_proj_dim > 0) {
        // M-CLIP's LinearTransformation (nn.Linear [E, w] with bias), transposed to the [w, E] text_head reads
        const std::vector<float> lin = to_host(param(m, "LinearTransformation.weight", E * w), (size_t)(E * w));
        std::vector<float> proj((size_t)(E * w));
        for (long long e = 0; e < E; ++e)
            for (long long i = 0; i < w; ++i) proj[(size_t)(i * E + e)] = lin[(size_t)(e * w + i)];
        T.proj = upload_derived(m, proj);
        m->raw.erase("LinearTransformation.weight");
        T.b_tproj = param(m, "LinearTransformation.bias", E);
    }
}

struct Counter {
    int n = 0;
};

// A GEMM (cls 0) or attention (cls 1) launch: launch() returns the number of kernels it launched, which is counted;
// while profiling, events bracket it for b200_model_profile.
template <class Launch>
void profiled(b200_model* m, Counter& c, int cls, Launch&& launch) {
    if (!m->profiling) {
        c.n += launch();
        return;
    }
    if ((size_t)(2 * m->prof_n + 2) > m->prof_ev.size()) {
        for (int i = 0; i < 64; ++i) m->prof_ev.push_back(make_event());
        m->prof_cls.resize(m->prof_ev.size() / 2);
    }
    m->prof_cls[m->prof_n] = cls;
    MB_CUDA(cudaEventRecord(m->prof_ev[2 * m->prof_n].get(), m->stream));
    c.n += launch();
    MB_CUDA(cudaEventRecord(m->prof_ev[2 * m->prof_n + 1].get(), m->stream));
    ++m->prof_n;
}

gemm::Epilogue epilogue(void* out, int ldo, const float* bias = nullptr, int act = gemm::ACT_NONE,
                        bool out_fp32 = false, const void* residual = nullptr, int ldr = 0) {
    gemm::Epilogue e;
    e.bias = bias;
    e.residual = residual;
    e.ldr = ldr;
    e.act = act;
    e.out = out;
    e.ldo = ldo;
    e.out_fp32 = out_fp32 ? 1 : 0;
    return e;
}

// out = ep(A[M, K] W[N, K]^T), A's rows lda elements apart (0: K)
void linear(b200_model* m, Counter& c, const __nv_bfloat16* A, int M, int K, const __nv_bfloat16* W, int N,
            const gemm::Epilogue& ep, int lda = 0) {
    profiled(m, c, 0, [&] {
        return gemm::launch(A, lda ? lda : K, W, M, N, K, ep, m->sms, m->stream) == gemm::KERNEL_NONE ? 0 : 1;
    });
}

// The transformer layers of a tower.  x (fp32) is the residual stream, h (bf16) the LayerNorm output the next GEMM
// consumes.  Pre-LN (open_clip ResidualAttentionBlock, timm's ViT and Eva Blocks): LN x -> h before the QKV and fc1
// GEMMs.  Post-LN (HF BertLayer, MPNetLayer with the tower's relative-position bias, NewModel): on entry x and h both
// hold the embedding LayerNorm output, and LN rewrites x in place (x -> x and h) after each residual GEMM.  A tower may
// rotate q and k after the QKV GEMM (T.rope), LayerNorm the attention output before the out-projection (EVA02's
// attn.norm) and run a gated MLP (Mlp).  A video tower (T.frames > 0, B = videos * frames) runs LanguageBind's temporal
// step first (modeling_video.py:209-232): x += temporal_embedding[t], then x += out_proj(attention over the frames of
// each token position (temporal_layer_norm1(x))).  Layers [first, first + count) run (count < 0: to the last one).
// MASK_CLS reads the sequences' token ids, cls_ids [B, S - 1].
void run_layers(b200_model* m, Counter& c, const TowerW& T, int B, int S, int mask_mode, int first = 0,
                int count = -1, const int32_t* cls_ids = nullptr) {
    const int M = B * S, w = T.d.width, aw = T.aw, mlp = T.d.mlp, fc1 = fc1_cols(T);
    const int end = count < 0 ? (int)T.layers.size() : first + count;
    float* x = m->x.get();
    __nv_bfloat16 *h = m->h.get(), *qkv = m->qkv.get(), *o = m->o.get(), *u = m->u.get();
    const int32_t* kv_len = mask_mode == attention::MASK_KEYLEN ? m->aux.get()
                            : mask_mode == attention::MASK_CLS  ? cls_ids
                                                                : nullptr;
    auto ln = [&](const float* g, const float* b) {
        c.n += kernels::layernorm(x, w, g, b, T.eps, M, w, T.pre_ln ? nullptr : x, h, m->stream);
    };
    for (int i = first; i < end; ++i) {
        const LayerW& L = T.layers[i];
        if (T.frames) {
            c.n += kernels::temporal_embed_ln(x, L.temb, S, T.frames, L.tln_w, L.tln_b, T.eps, M, w, h, m->stream);
            linear(m, c, h, M, w, L.w_tqkv, 3 * w, epilogue(qkv, 3 * w, L.b_tqkv));
            profiled(m, c, 1, [&] {
                return kernels::temporal_attention(qkv, B / T.frames, T.frames, S, w, T.d.heads, o, m->stream);
            });
            linear(m, c, o, M, w, L.w_to, w, epilogue(x, w, L.b_to, gemm::ACT_NONE, true, x, w));
        }
        if (T.pre_ln) ln(L.ln1_w, L.ln1_b);
        linear(m, c, h, M, w, L.w_qkv, 3 * aw, epilogue(qkv, 3 * aw, L.b_qkv));
        if (T.rope) c.n += kernels::rope_qk(qkv, B, S, T.rope_first, aw, T.rope, T.rope_pairing, m->stream);
        profiled(m, c, 1, [&] {
            return attention::launch(qkv, o, B, S, aw, T.d.heads, mask_mode, kv_len, T.rel_bias, m->stream,
                                     w / T.d.heads);
        });
        if (L.ln_attn_w) c.n += kernels::layernorm_bf16(o, w, L.ln_attn_w, L.ln_attn_b, T.eps, M, w, h, m->stream);
        linear(m, c, L.ln_attn_w ? h : o, M, aw, L.w_o, w, epilogue(x, w, L.b_o, gemm::ACT_NONE, true, x, w));
        ln(T.pre_ln ? L.ln2_w : L.ln1_w, T.pre_ln ? L.ln2_b : L.ln1_b);
        linear(m, c, h, M, w, L.w_fc, fc1,
               epilogue(u, fc1, L.b_fc, T.mlp_form == Mlp::ACT ? T.act : gemm::ACT_NONE));
        if (T.mlp_form == Mlp::SWIGLU_LN)
            c.n += kernels::swiglu_ln(u, M, mlp, T.mlp_h, L.ln_mlp_w, L.ln_mlp_b, T.eps, u, fc1, m->stream);
        else if (T.mlp_form == Mlp::GEGLU)
            c.n += kernels::geglu(u, M, mlp, u, fc1, m->stream);
        linear(m, c, u, M, mlp, L.w_proj, w, epilogue(x, w, L.b_proj, gemm::ACT_NONE, true, x, w), fc1);
        if (!T.pre_ln) ln(L.ln2_w, L.ln2_b);
    }
}

// One folded ResNet conv over n images of H x H output pixels (NHWC bf16 x -> out): bias, then ReLU with the optional
// bf16 residual added before it, or neither.  The stem conv (cin 3) takes stem_im2col's rows as x.
void resnet_conv(b200_model* m, Counter& c, const ConvW& cw, const __nv_bfloat16* x, int n, int H,
                 const __nv_bfloat16* residual, bool relu, __nv_bfloat16* out) {
    const gemm::Epilogue e =
        epilogue(out, cw.cout, cw.b, relu ? gemm::ACT_RELU : gemm::ACT_NONE, false, residual, cw.cout);
    profiled(m, c, 0, [&] { return gemm::launch_conv(x, n, H, H, cw.cin, cw.k, cw.w, cw.cout, e, m->sms, m->stream); });
}

// The ResNet CLIP image tower over n images (uint8 HWC u8 or normalised fp32 CHW f32, at the model's size): buffers
// A B C D rotate so that every block starts and ends in A.
void forward_resnet(b200_model* m, Counter& c, const uint8_t* u8, const float* f32, int n, int normalize, float* d_out) {
    ResnetW& R = m->resnet;
    const b200_model_desc& d = m->desc;
    __nv_bfloat16 *A = R.buf[0].get(), *B = R.buf[1].get(), *Cb = R.buf[2].get(), *D = R.buf[3].get();
    const int S = d.resnet_image_size, width = d.resnet_width;
    int H = S / 2;
    c.n += kernels::stem_im2col(u8, f32, n, S, d.image_mean, d.image_std, B, m->stream);
    resnet_conv(m, c, R.stem[0], B, n, H, nullptr, true, Cb);
    resnet_conv(m, c, R.stem[1], Cb, n, H, nullptr, true, D);
    resnet_conv(m, c, R.stem[2], D, n, H, nullptr, true, Cb);
    c.n += kernels::avgpool2_nhwc(Cb, n, H, H, width, A, m->stream);
    H /= 2;
    for (const BottleneckW& blk : R.blocks) {
        resnet_conv(m, c, blk.c1, A, n, H, nullptr, true, B);
        resnet_conv(m, c, blk.c2, B, n, H, nullptr, true, Cb);
        const __nv_bfloat16 *main = Cb, *identity = A;
        if (blk.stride > 1) {
            c.n += kernels::avgpool2_nhwc(Cb, n, H, H, blk.c2.cout, B, m->stream);
            c.n += kernels::avgpool2_nhwc(A, n, H, H, blk.c1.cin, Cb, m->stream);
            H /= 2;
            main = B;
            resnet_conv(m, c, blk.ds, Cb, n, H, nullptr, false, D);
            identity = D;
        } else if (blk.has_ds) {
            resnet_conv(m, c, blk.ds, A, n, H, nullptr, false, D);
            identity = D;
        }
        // in place over the identity when it is A: a tile reads the residual rows and columns it writes, nothing else
        resnet_conv(m, c, blk.c3, main, n, H, identity, true, A);
    }
    // attention pool: tokens [mean; pixels] + pos -> B; K|V of every token -> Cb; q of token 0 (rows T C apart) -> D;
    // one query per image and head -> A; c_proj -> pooled; L2
    const int C = R.C, HW = R.grid * R.grid, T = HW + 1, E = d.embed_dim;
    c.n += kernels::attnpool_tokens(A, R.pos, n, HW, C, B, m->stream);
    float* q = reinterpret_cast<float*>(D);
    linear(m, c, B, n * T, C, R.w_kv, 2 * C, epilogue(Cb, 2 * C, R.b_kv));
    linear(m, c, B, n, C, R.w_q, C, epilogue(q, C, R.b_q, gemm::ACT_NONE, true), T * C);
    profiled(m, c, 1, [&] { return kernels::map_attention(q, C, Cb, n, T, C, d.resnet_heads, A, m->stream); });
    linear(m, c, A, n, C, R.w_c, E, epilogue(m->pooled.get(), E, R.b_c, gemm::ACT_NONE, true));
    c.n += kernels::l2_rows(m->pooled.get(), n, E, normalize, d_out, m->stream);
}

// The patch conv of T (no bias in its weights) over n images (device uint8 [n, S, S, 3] u8, or device fp32 CHW f32)
// through epilogue e, into the n * T.tokens token rows.
void patch_embed(b200_model* m, Counter& c, const TowerW& T, const uint8_t* u8, const float* f32, int n,
                 const gemm::Epilogue& e) {
    const int S = T.d.image_size, p = T.d.patch, w = T.d.width;
    if (u8) {
        // uint8 pixels -> ToTensor + Normalize -> bf16 inside the GEMM's operand load: no patch matrix in HBM
        gemm::PatchGather pg;
        pg.img = u8;
        pg.n = n;
        pg.S = S;
        pg.patch = p;
        pg.cls = T.cls_rows;
        for (int i = 0; i < 3; ++i) {
            pg.mean[i] = m->desc.image_mean[i];
            pg.std[i] = m->desc.image_std[i];
        }
        profiled(m, c, 0, [&] { return gemm::launch_patch_embed(pg, T.conv_wg, w, e, m->stream); });
    } else {
        // preprocessed fp32 CHW tensors (the reference's parity path)
        if (!m->patches)
            m->patches =
                DeviceBuffer<__nv_bfloat16>((size_t)m->desc.max_batch * std::max(1, T.frames) * T.tokens * T.kpad);
        c.n += kernels::im2col_f32(f32, n, S, p, T.kpad, T.cls_rows, m->patches.get(), m->stream);
        linear(m, c, m->patches.get(), n * T.tokens, T.kpad, T.conv_w, w, e);
    }
}

// A ViT trunk over n images (device uint8 [n, S, S, 3] u8, or device fp32 CHW f32): patch embedding, ln_pre (CLIP) and
// the layers, leaving the n * T.tokens token rows in x.  A video tower's images are the frames of n / T.frames videos.
void forward_vit(b200_model* m, Counter& c, const TowerW& T, const uint8_t* u8, const float* f32, int n) {
    const int w = T.d.width, per = std::max(1, T.frames);
    float* x = m->x.get();
    // x = positional embedding (+ class embedding on each image's first row), then conv1 (no bias) of every token row
    // added onto it in place; a class-token row multiplies a zero A row.  SigLIP has no class row; its conv bias, and
    // EVA02's, is already in T.pos; a video tower's T.pos spans a video's frames, class rows included.
    c.n += kernels::vit_embed_rows(x, T.cls, T.pos, n / per, per * T.tokens, w, m->stream);
    patch_embed(m, c, T, u8, f32, n, epilogue(x, w, nullptr, gemm::ACT_NONE, true, x, w));
    if (T.ln_pre_w)
        c.n += kernels::layernorm(x, w, T.ln_pre_w, T.ln_pre_b, T.eps, n * T.tokens, w, x, nullptr, m->stream);
    run_layers(m, c, T, n, T.tokens, attention::MASK_NONE);
}

// SigLIP vision head over the n * S token rows in x: final LayerNorm of every token -> h, K|V projection -> qkv
// [n * S, 2w], one latent query per head attending over its image's tokens -> o [n, w], then proj -> pooled (fp32),
// pooled + MLP(LN(pooled)), optional L2 -> d_out.
void map_head(b200_model* m, Counter& c, const TowerW& T, int n, int normalize, float* d_out) {
    const int S = T.tokens, w = T.d.width, M = n * S;
    const MapW& P = T.map;
    float* pooled = m->pooled.get();
    c.n += kernels::layernorm(m->x.get(), w, T.ln_out_w, T.ln_out_b, T.eps, M, w, nullptr, m->h.get(), m->stream);
    linear(m, c, m->h.get(), M, w, P.w_kv, 2 * w, epilogue(m->qkv.get(), 2 * w, P.b_kv));
    __nv_bfloat16* o = m->o.get();
    profiled(m, c, 1, [&] { return kernels::map_attention(P.q, 0, m->qkv.get(), n, S, w, T.d.heads, o, m->stream); });
    linear(m, c, o, n, w, P.w_proj, w, epilogue(pooled, w, P.b_proj, gemm::ACT_NONE, true));
    c.n += kernels::layernorm(pooled, w, P.ln_w, P.ln_b, T.eps, n, w, nullptr, m->h.get(), m->stream);
    linear(m, c, m->h.get(), n, w, P.w_fc1, P.mlp, epilogue(m->u.get(), P.mlp, P.b_fc1, gemm::ACT_GELU));
    linear(m, c, m->u.get(), n, P.mlp, P.w_fc2, w, epilogue(pooled, w, P.b_fc2, gemm::ACT_NONE, true, pooled, w));
    c.n += kernels::l2_rows(pooled, n, w, normalize, d_out, m->stream);
}

// CoCa's attentional pooler over the n * S token rows in x (TowerW::map): ln_k of every token -> h, K|V -> qkv
// [n * S, 2d], query 0's heads attending over its image's tokens -> o [n, d], out_proj -> x [n, d] (fp32; the trunk's
// rows are no longer read), then ln_post, proj and the unit normalisation of every CoCa output -> d_out.
void coca_pool_head(b200_model* m, Counter& c, const TowerW& T, int n, int normalize, float* d_out) {
    const int S = T.tokens, w = T.d.width, M = n * S, d = m->desc.embed_dim;
    const MapW& P = T.map;
    c.n += kernels::layernorm(m->x.get(), w, P.ln_w, P.ln_b, T.eps, M, w, nullptr, m->h.get(), m->stream);
    linear(m, c, m->h.get(), M, w, P.w_kv, 2 * d, epilogue(m->qkv.get(), 2 * d, P.b_kv));
    __nv_bfloat16* o = m->o.get();
    profiled(m, c, 1, [&] {
        return kernels::map_attention(P.q, 0, m->qkv.get(), n, S, d, m->desc.attn_pool_heads, o, m->stream);
    });
    linear(m, c, o, n, d, P.w_proj, d, epilogue(m->x.get(), d, P.b_proj, gemm::ACT_NONE, true));
    c.n += kernels::clip_head(m->x.get(), 1, nullptr, T.ln_out_w, T.ln_out_b, T.eps, T.proj, n, d, d, normalize, d_out,
                              m->pooled.get(), m->stream, true);
}

// The ConvNeXt CLIP image tower over n images (device uint8 HWC u8 or normalised fp32 CHW f32, at the model's size).
void forward_convnext(b200_model* m, Counter& c, const uint8_t* u8, const float* f32, int n, int normalize,
                      float* d_out) {
    const ConvnextW& X = m->convnext;
    const TowerW& T = m->vision;
    const b200_model_desc& d = m->desc;
    const float eps = d.layer_norm_eps;
    const int E = d.embed_dim, C0 = T.d.width;
    float* x = X.x.get();
    __nv_bfloat16 *h = X.h.get(), *u = X.u.get();
    // stem: the 4 x 4 stride-4 conv with its bias -> x, then its LayerNorm in place: the residual stream
    patch_embed(m, c, T, u8, f32, n, epilogue(x, C0, X.stem_b, gemm::ACT_NONE, true));
    int H = T.grid;
    c.n += kernels::ln_pixels(x, n, H, H, C0, X.stem_ln_w, X.stem_ln_b, eps, x, nullptr, m->stream);
    int prev = C0;
    for (const ConvnextStageW& st : X.stages) {
        const int C = st.C;
        if (st.ds_w) {
            // LayerNorm + 2 x 2 patches -> h; the GEMM reads only h, so it may overwrite x
            c.n += kernels::ln_pixels(x, n, H, H, prev, st.ds_ln_w, st.ds_ln_b, eps, nullptr, h, m->stream);
            H /= 2;
            linear(m, c, h, n * H * H, 4 * prev, st.ds_w, C, epilogue(x, C, st.ds_b, gemm::ACT_NONE, true));
        }
        const int M = n * H * H;
        for (const ConvnextBlockW& B : st.blocks) {
            c.n += kernels::dwconv7_ln(x, n, H, H, C, B.dw_w, B.dw_b, B.ln_w, B.ln_b, eps, h, m->stream);
            linear(m, c, h, M, C, B.w1, 4 * C, epilogue(u, 4 * C, B.b1, gemm::ACT_GELU));
            linear(m, c, u, M, 4 * C, B.w2, C, epilogue(x, C, B.b2, gemm::ACT_NONE, true, x, C));
        }
        prev = C;
    }
    // head: mean over the pixels + LayerNorm -> h [n, C3], then the projection or the MLP -> pooled, L2
    float* pooled = m->pooled.get();
    c.n += kernels::pool_ln(x, n, H * H, prev, X.head_ln_w, X.head_ln_b, eps, h, m->stream);
    if (X.w_proj) {
        linear(m, c, h, n, prev, X.w_proj, E, epilogue(pooled, E, nullptr, gemm::ACT_NONE, true));
    } else {
        linear(m, c, h, n, prev, X.w_fc1, 2 * E, epilogue(u, 2 * E, X.b_fc1, gemm::ACT_GELU));
        linear(m, c, u, n, 2 * E, X.w_fc2, E, epilogue(pooled, E, nullptr, gemm::ACT_NONE, true));
    }
    c.n += kernels::l2_rows(pooled, n, E, normalize, d_out, m->stream);
}

// images already as device uint8 [n, S, S, 3] (u8 != nullptr) or device fp32 CHW (f32 != nullptr)
void forward_images_eager(b200_model* m, Counter& c, const uint8_t* u8, const float* f32, int n, int normalize,
                          float* d_out) {
    const TowerW& T = m->vision;
    switch (m->kind.vision) {
    case VisionKind::CLIP_VIT:
        forward_vit(m, c, T, u8, f32, n);
        c.n += kernels::clip_head(m->x.get(), T.tokens, nullptr, T.ln_out_w, T.ln_out_b, T.eps, T.proj, n, T.d.width,
                                  m->desc.embed_dim, normalize, d_out, m->pooled.get(), m->stream);
        break;
    case VisionKind::SIGLIP_VIT:
        forward_vit(m, c, T, u8, f32, n);
        map_head(m, c, T, n, normalize, d_out);
        break;
    case VisionKind::COCA_VIT:
        forward_vit(m, c, T, u8, f32, n);
        coca_pool_head(m, c, T, n, normalize, d_out);
        break;
    case VisionKind::RESNET:
        forward_resnet(m, c, u8, f32, n, normalize, d_out);
        break;
    case VisionKind::CONVNEXT:
        forward_convnext(m, c, u8, f32, n, normalize, d_out);
        break;
    case VisionKind::EVA_VIT: {
        // trunk.norm of each image's class row (rows T.tokens apart) -> h [n, w], the head Linear with its bias, L2
        const int w = T.d.width, E = m->desc.embed_dim;
        forward_vit(m, c, T, u8, f32, n);
        c.n += kernels::layernorm(m->x.get(), (long long)T.tokens * w, T.ln_out_w, T.ln_out_b, T.eps, n, w, nullptr,
                                  m->h.get(), m->stream);
        linear(m, c, m->h.get(), n, w, T.w_tproj, E, epilogue(m->pooled.get(), E, T.b_tproj, gemm::ACT_NONE, true));
        c.n += kernels::l2_rows(m->pooled.get(), n, E, normalize, d_out, m->stream);
        break;
    }
    }
}

// OWL-ViT's detection over n images (device uint8 [n, S, S, 3]) and the query's text embedding t [E] (device): the
// trunk's rows in x; the merged patch features -> h; the class head GEMM -> x (fp32 [M, ncls], the trunk's rows are
// no longer read) and the logits; box_head dense0 -> u, dense1 -> o, then dense2 and the box bias -> boxes.
void forward_detect_eager(b200_model* m, Counter& c, const uint8_t* u8, int n, const float* t, float* logits,
                          float* boxes) {
    const TowerW& T = m->vision;
    const OwlW& D = m->owl;
    const int w = T.d.width, P = T.grid * T.grid, M = n * P;
    float* x = m->x.get();
    __nv_bfloat16 *h = m->h.get(), *u = m->u.get(), *o = m->o.get();
    forward_vit(m, c, T, u8, nullptr, n);
    c.n += kernels::owl_merge_ln(x, n, T.tokens, w, T.ln_out_w, T.ln_out_b, D.ln_w, D.ln_b, T.eps, h, m->stream);
    linear(m, c, h, M, w, D.w_cls, D.ncls, epilogue(x, D.ncls, D.b_cls, gemm::ACT_NONE, true));
    c.n += kernels::owl_class_logits(x, D.ncls, M, m->desc.embed_dim, t, logits, m->stream);
    linear(m, c, h, M, w, D.w_box0, w, epilogue(u, w, D.b_box0, gemm::ACT_GELU));
    linear(m, c, u, M, w, D.w_box1, w, epilogue(o, w, D.b_box1, gemm::ACT_GELU));
    c.n += kernels::owl_boxes(o, M, w, P, D.w_box2, D.b_box2, D.box_bias, boxes, m->stream);
}

// d_types: token-type ids [n, S] of a classifier (NULL: all 0); normalize is then the classifier's activation (0
// identity, 1 sigmoid)
void forward_tokens_eager(b200_model* m, Counter& c, const int32_t* d_ids, const int32_t* d_mask, const int32_t* d_types,
                          int n, int S, int normalize, float* d_out) {
    const TowerW& T = m->text;
    const int w = T.d.width, E = m->desc.embed_dim;
    float* x = m->x.get();
    int32_t* aux = m->aux.get();
    switch (m->kind.text) {
    case TextKind::CLIP:
        // causal layers; ln_final of each sequence's eot row, projection, optional L2 (LanguageBind: always L2, then
        // optionally once more)
        c.n += kernels::clip_text_embed(d_ids, T.tok, T.pos, n, S, w, T.d.vocab, x, aux, m->stream);
        run_layers(m, c, T, n, S, attention::MASK_CAUSAL);
        if (m->desc.video_frames)
            c.n += kernels::frame_mean_head(x, S, 1, aux, T.ln_out_w, T.ln_out_b, T.eps, T.proj, n, w, E, 1.f, normalize,
                                            d_out, m->pooled.get(), m->stream);
        else
            c.n += kernels::clip_head(x, S, aux, T.ln_out_w, T.ln_out_b, T.eps, T.proj, n, w, E, normalize, d_out,
                                      m->pooled.get(), m->stream);
        break;
    case TextKind::COCA: {
        // ids [n, S]; the CLS row appended after them is the last of St token rows, pooled (aux = St - 1) through
        // ln_final and the projection, then the unit normalisation
        const int St = S + 1;
        c.n += kernels::clip_text_embed(d_ids, T.tok, T.pos, n, St, w, T.d.vocab, x, aux, m->stream, T.text_cls);
        run_layers(m, c, T, n, St, attention::MASK_CLS, 0, -1, d_ids);
        c.n += kernels::clip_head(x, St, aux, T.ln_out_w, T.ln_out_b, T.eps, T.proj, n, w, E, normalize, d_out,
                                  m->pooled.get(), m->stream, true);
        break;
    }
    case TextKind::SIGLIP:
        // bidirectional layers; ln_final of each sequence's last row (stride S rows) -> h [n, w], biased projection
        c.n += kernels::clip_text_embed(d_ids, T.tok, T.pos, n, S, w, T.d.vocab, x, aux, m->stream);
        run_layers(m, c, T, n, S, attention::MASK_NONE);
        c.n += kernels::layernorm(x + (size_t)(S - 1) * w, (long long)S * w, T.ln_out_w, T.ln_out_b, T.eps, n, w,
                                  nullptr, m->h.get(), m->stream);
        linear(m, c, m->h.get(), n, w, T.w_tproj, E, epilogue(m->pooled.get(), E, T.b_tproj, gemm::ACT_NONE, true));
        c.n += kernels::l2_rows(m->pooled.get(), n, E, normalize, d_out, m->stream);
        break;
    case TextKind::BERT:
    case TextKind::ROBERTA:
    case TextKind::GTE:
        // RoBERTa position ids count from pad_id; XLM-R also adds its single token-type row (T.type0 is NULL for
        // MPNet); GTE has no position table (T.pos is NULL)
        if (m->kind.text != TextKind::ROBERTA)
            c.n += kernels::bert_embed_ln(d_ids, d_mask, T.tok, T.pos, T.type0, T.emb_ln_w, T.emb_ln_b, T.eps, n, S, w,
                                          T.d.vocab, x, m->h.get(), aux, m->stream, d_types,
                                          std::max(1, m->desc.type_vocab));
        else
            c.n += kernels::roberta_embed_ln(d_ids, d_mask, T.tok, T.pos, T.type0, T.emb_ln_w, T.emb_ln_b, T.eps, n, S,
                                             w, T.d.vocab, m->desc.pad_id, x, m->h.get(), aux, m->stream);
        run_layers(m, c, T, n, S, attention::MASK_KEYLEN);
        if (T.cls_w)   // BertForSequenceClassification: pooler, classifier, activation
            c.n += kernels::cls_head(x, S, n, w, T.pool_w, T.pool_b, T.cls_w, T.cls_b, E, normalize, d_out, m->stream);
        else if (T.proj)   // M-CLIP: the masked mean, projected
            c.n += kernels::text_head(x, aux, n, S, w, T.proj, T.b_tproj, E, normalize, d_out, m->pooled.get(),
                                      m->stream);
        else
            c.n += kernels::bert_head(x, aux, n, S, w, m->desc.pool, normalize, d_out, m->stream);
        break;
    }
}

// Small batches (a single query, a handful of chunks) are launch-bound: ~90-180 kernels of a few microseconds each,
// every GEMM launch also encoding two tensor maps on the host.  The first call of a shape runs eagerly (one-time
// attribute set-up happens there), the second is captured into a CUDA graph, later ones replay it.
constexpr long long GRAPH_MAX_TOKENS = 8192;
constexpr size_t GRAPH_MAX_ENTRIES = 64;

template <class Body>
void run_graphed(b200_model* m, Counter& c, const b200_model::GraphKey& key, long long tokens, Body&& body) {
    static const bool disabled = getenv("MARQO_B200_NO_GRAPHS") != nullptr;   // kill switch / A-B timing
    if (disabled || tokens > GRAPH_MAX_TOKENS || m->profiling || m->external_stream) {
        body(c);
        return;
    }
    auto it = m->graphs.find(key);
    if (it == m->graphs.end()) {
        if (m->graphs.size() < GRAPH_MAX_ENTRIES) m->graphs[key] = b200_model::GraphEntry{};
        body(c);
        return;
    }
    if (!it->second.exec) {
        Counter cc;
        MB_CUDA(cudaStreamBeginCapture(m->stream, cudaStreamCaptureModeThreadLocal));
        cudaGraph_t graph = nullptr;
        try {
            body(cc);
        } catch (...) {
            cudaStreamEndCapture(m->stream, &graph);
            if (graph) cudaGraphDestroy(graph);
            m->graphs.erase(it);
            throw;
        }
        MB_CUDA(cudaStreamEndCapture(m->stream, &graph));
        cudaGraphExec_t exec = nullptr;
        const cudaError_t e = cudaGraphInstantiate(&exec, graph, 0);
        cudaGraphDestroy(graph);
        MB_CUDA(e);
        it->second.exec.reset(exec);
        it->second.launches = cc.n;
    }
    MB_CUDA(cudaGraphLaunch(it->second.exec.get(), m->stream));
    c.n += it->second.launches;
}

void forward_images(b200_model* m, Counter& c, const uint8_t* u8, const float* f32, int n, int normalize, float* d_out) {
    const b200_model::GraphKey key{Call::IMAGES, n, 0, normalize, u8, f32, d_out};
    run_graphed(m, c, key, (long long)n * m->vision.tokens,
                [&](Counter& cc) { forward_images_eager(m, cc, u8, f32, n, normalize, d_out); });
}

void forward_tokens(b200_model* m, Counter& c, const int32_t* d_ids, const int32_t* d_mask, const int32_t* d_types, int n,
                    int S, int normalize, float* d_out) {
    const b200_model::GraphKey key{Call::TOKENS, n, S, normalize, d_ids, d_mask, d_out, d_types};
    run_graphed(m, c, key, (long long)n * S,
                [&](Counter& cc) { forward_tokens_eager(m, cc, d_ids, d_mask, d_types, n, S, normalize, d_out); });
}

void forward_detect(b200_model* m, Counter& c, const uint8_t* u8, int n, const float* t, float* logits, float* boxes) {
    const b200_model::GraphKey key{Call::DETECT, n, 0, 0, u8, t, logits, boxes};
    run_graphed(m, c, key, (long long)n * m->vision.tokens,
                [&](Counter& cc) { forward_detect_eager(m, cc, u8, n, t, logits, boxes); });
}

// n videos of T.frames transformed frames each (device fp32 CHW [n * frames, 3, S, S]): the trunk, then LanguageBind's
// head (the mean of the frames' ln_post class rows, visual.proj, L2 times exp(logit_scale), optional L2)
void forward_videos(b200_model* m, Counter& c, const float* f32, int n, int normalize, float* d_out) {
    const TowerW& T = m->vision;
    const b200_model::GraphKey key{Call::VIDEOS, n, 0, normalize, nullptr, f32, d_out};
    run_graphed(m, c, key, (long long)n * T.frames * T.tokens, [&](Counter& cc) {
        forward_vit(m, cc, T, nullptr, f32, n * T.frames);
        cc.n += kernels::frame_mean_head(m->x.get(), T.tokens, T.frames, nullptr, T.ln_out_w, T.ln_out_b, T.eps, T.proj,
                                         n, T.d.width, m->desc.embed_dim, T.out_scale, normalize, d_out,
                                         m->pooled.get(), m->stream);
    });
}

void require_ready(b200_model* m) {
    MB_CHECK_ARG(m != nullptr, "model is NULL");
    if (!m->finalized) fail(B200_ERR_INVALID_ARG, "b200_model_finalize has not been called");
}

// Which calls a model takes: an OWL-ViT detector only detects, a video model encodes videos (and its text), and a text
// tower with a classification head classifies instead of encoding.
void require_accepts(b200_model* m, Call call) {
    const VisionKind vk = m->kind.vision;
    const char* owl = "this model is an OWL-ViT detector: detect images with a query";
    switch (call) {
    case Call::IMAGES:
        MB_CHECK_ARG(vk != VisionKind::NONE, "this model has no vision tower");
        MB_CHECK_ARG(!m->desc.owl_detect, "%s", owl);
        MB_CHECK_ARG(vk != VisionKind::VIDEO_VIT, "this model is a video model: encode videos of %d frames",
                     m->vision.frames);
        break;
    case Call::TOKENS:
    case Call::CLASSIFY:
        MB_CHECK_ARG(m->kind.text != TextKind::NONE, "this model has no text tower");
        MB_CHECK_ARG(!m->desc.owl_detect, "%s", owl);
        if (call == Call::CLASSIFY)
            MB_CHECK_ARG(m->desc.cls_labels > 0, "this model has no classification head (cls_labels 0)");
        else
            MB_CHECK_ARG(m->desc.cls_labels == 0, "this model is a classifier (cls_labels %d): classify its tokens",
                         m->desc.cls_labels);
        break;
    case Call::DETECT:
        MB_CHECK_ARG(m->desc.owl_detect, "this model has no OWL-ViT detection head (owl_detect 0)");
        break;
    case Call::VIDEOS:
        MB_CHECK_ARG(vk == VisionKind::VIDEO_VIT, "this model has no video tower (video_frames 0)");
        break;
    }
}

// Every model call.  All its refusals come first, so that a refused call writes nothing and leaves last_timing as it
// was: readiness, whether the model takes `call`, then `check`, the call's own argument checks, which returns the bytes
// of host input the call stages in in_dev (0 for device inputs).  Then, under the model's lock on its device, in_dev
// is sized and `body` runs on the model's stream, timed into last_timing, with a final synchronise if `sync`.
template <class Check, class Body>
int model_call(b200_model* m, Call call, int sync, Check&& check, Body&& body) {
    return guarded([&] {
        require_ready(m);
        require_accepts(m, call);
        const size_t staged = check();
        std::lock_guard<std::mutex> lk(m->mu);
        DeviceGuard g(m->device);
        if (staged > m->in_dev.size()) m->in_dev = DeviceBuffer<uint8_t>(staged);
        Counter c;
        MB_CUDA(cudaEventRecord(m->ev0.get(), m->stream));
        body(c);
        MB_CUDA(cudaEventRecord(m->ev1.get(), m->stream));
        m->timing_valid = true;
        m->last_launches = c.n;
        if (sync) MB_CUDA(cudaStreamSynchronize(m->stream));
    });
}

void to_device(b200_model* m, void* dst, const void* src, size_t bytes) {
    MB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, m->stream));
}

// A device output of a host call and where it goes: `per` floats of each item.
struct HostOut {
    float* host;
    const float* dev;
    size_t per;
};

// A host call's n items in sub-batches of up to cap: stage(o, nb) copies the inputs of items o .. o + nb - 1 into
// in_dev, run(o, nb) runs the device path over them, and every output's nb items come back before the synchronise
// that frees in_dev for the next sub-batch.
template <class Stage, class Run>
void host_batches(b200_model* m, int n, int cap, Stage&& stage, Run&& run, std::initializer_list<HostOut> outs) {
    for (int o = 0; o < n; o += cap) {
        const int nb = std::min(cap, n - o);
        stage(o, nb);
        run(o, nb);
        for (const HostOut& r : outs)
            MB_CUDA(cudaMemcpyAsync(r.host + (size_t)o * r.per, r.dev, (size_t)nb * r.per * sizeof(float),
                                    cudaMemcpyDeviceToHost, m->stream));
        MB_CUDA(cudaStreamSynchronize(m->stream));
    }
}

// the n, h, w and buffers of a uint8 image or video call
void check_u8_args(bool buffers, int n, int h, int w) {
    MB_CHECK_ARG(buffers, "NULL buffer");
    MB_CHECK_ARG(n > 0 && h > 0 && w > 0, "n, h, w must be positive");
}

int batch_cap_tokens(b200_model* m, int tokens_per_item) {
    return (int)std::max<long long>(1, std::min<long long>(m->desc.max_batch, m->max_tokens / tokens_per_item));
}

// images per forward pass: what the image tower's activation buffers hold
int image_batch_cap(b200_model* m) {
    return m->kind.vision == VisionKind::CONVNEXT ? m->convnext.max_images : batch_cap_tokens(m, m->vision.tokens);
}

// videos per forward pass: what the workspaces hold
int video_batch_cap(b200_model* m) { return batch_cap_tokens(m, m->vision.frames * m->vision.tokens); }

// device-resident uint8 videos [n, frames, h, w, 3] -> embeddings: each sub-batch's frames transformed into video_f32,
// then one forward pass
void encode_videos_u8_dev(b200_model* m, Counter& c, const uint8_t* d_vid, int n, int h, int w, int normalize,
                          float* d_out) {
    const TowerW& T = m->vision;
    const int cap = video_batch_cap(m), F = T.frames;
    for (int o = 0; o < n; o += cap) {
        const int nb = std::min(cap, n - o);
        c.n += kernels::video_resize_crop(d_vid + (size_t)o * F * h * w * 3, (long long)nb * F, h, w, T.d.image_size,
                                          m->desc.image_mean, m->desc.image_std, m->video_f32.get(), m->stream);
        forward_videos(m, c, m->video_f32.get(), nb, normalize, d_out + (size_t)o * m->desc.embed_dim);
    }
}

// open_clip's SigLIP and DFN5B preprocessing squashes (no crop); every other tower crops
bool resize_squashes(b200_model* m) { return m->kind.vision == VisionKind::SIGLIP_VIT || m->desc.resize_squash; }

// nb device uint8 images of h x w as the image tower takes them, S x S: resized into m->resized, unless already S x S
const uint8_t* resize_images(b200_model* m, Counter& c, const uint8_t* src, int nb, int h, int w) {
    const int S = m->vision.d.image_size;
    if (h == S && w == S) return src;
    if (resize_squashes(m))
        c.n += kernels::resize_squash_u8(src, nb, h, w, S, m->resized.get(), m->stream);
    else
        c.n += kernels::resize_crop_u8(src, nb, h, w, S, m->resized.get(), m->stream);
    return m->resized.get();
}

// device-resident uint8 images of size h x w -> embeddings
void encode_images_u8_dev(b200_model* m, Counter& c, const uint8_t* d_img, int n, int h, int w, int normalize,
                          float* d_out) {
    const int cap = image_batch_cap(m);
    for (int o = 0; o < n; o += cap) {
        const int nb = std::min(cap, n - o);
        forward_images(m, c, resize_images(m, c, d_img + (size_t)o * h * w * 3, nb, h, w), nullptr, nb, normalize,
                       d_out + (size_t)o * m->desc.embed_dim);
    }
}

// device-resident uint8 images of any sizes (d_img, h, w: host arrays of n) -> embeddings: each sub-batch is resized
// into m->resized in one kernel pair, images already S x S included (their taps are the identity)
void encode_images_u8_ragged_dev(b200_model* m, Counter& c, const uint8_t* const* d_img, const int32_t* h,
                                 const int32_t* w, int n, int normalize, float* d_out) {
    const int S = m->vision.d.image_size;
    const int cap = image_batch_cap(m);
    for (int o = 0; o < n; o += cap) {
        const int nb = std::min(cap, n - o);
        c.n += kernels::resize_u8(d_img + o, h + o, w + o, nb, S, resize_squashes(m), m->resized.get(), m->stream);
        forward_images(m, c, m->resized.get(), nullptr, nb, normalize, d_out + (size_t)o * m->desc.embed_dim);
    }
}

// the arguments of a ragged image call, all checked before anything is written
void check_ragged_args(const uint8_t* const* imgs, const int32_t* h, const int32_t* w, int n) {
    MB_CHECK_ARG(imgs && h && w, "NULL array");
    MB_CHECK_ARG(n > 0, "n must be positive");
    for (int i = 0; i < n; ++i) {
        MB_CHECK_ARG(imgs[i] != nullptr, "image %d is NULL", i);
        MB_CHECK_ARG(h[i] > 0 && w[i] > 0, "image %d: height %d and width %d must be positive", i, h[i], w[i]);
    }
}

// The token rows a sequence of `seq` ids takes in the workspaces: CoCa's text tower appends its CLS row.
int token_rows(b200_model* m, int seq) { return m->kind.text == TextKind::COCA ? seq + 1 : seq; }

void encode_tokens_dev(b200_model* m, Counter& c, const int32_t* d_ids, const int32_t* d_mask, const int32_t* d_types,
                       int n, int S, int normalize, float* d_out) {
    const int cap = batch_cap_tokens(m, token_rows(m, S));
    for (int o = 0; o < n; o += cap) {
        const int nb = std::min(cap, n - o);
        forward_tokens(m, c, d_ids + (size_t)o * S, d_mask ? d_mask + (size_t)o * S : nullptr,
                       d_types ? d_types + (size_t)o * S : nullptr, nb, S, normalize,
                       d_out + (size_t)o * m->desc.embed_dim);
    }
}

// the arguments of a token call
void check_tokens_args(b200_model* m, int n, int S) {
    MB_CHECK_ARG(n > 0, "n must be positive");
    MB_CHECK_ARG(S > 0 && S <= m->text.tokens, "sequence length %d out of range (1..%d)", S, m->text.tokens);
    if (m->kind.text == TextKind::COCA)   // open_clip's CoCa tokenizer pads every text to ctx - 1 ids
        MB_CHECK_ARG(S == m->text.tokens - 1, "CoCa text: ids must be %d wide (got %d)", m->text.tokens - 1, S);
}

// The kernels implement prefix (right-padded) masks, which is what the tokenizer call at hugging_face_model.py:179-185
// produces.
void check_prefix_mask(const int32_t* mask, int n, int seq) {
    for (int b = 0; b < n; ++b) {
        bool seen_zero = false;
        for (int s = 0; s < seq; ++s) {
            const bool on = mask[(size_t)b * seq + s] != 0;
            if (on && seen_zero) fail(B200_ERR_UNSUPPORTED, "attention mask of item %d is not a prefix mask", b);
            seen_zero |= !on;
        }
    }
}

// b200_model_encode_tokens and b200_model_classify_tokens: host ids, mask and token types (either may be NULL) in
// sub-batches through in_dev; `normalize` is the classifier's activation for CLASSIFY
int tokens_host(b200_model* m, Call call, const int32_t* ids, const int32_t* attn_mask, const int32_t* types, int n,
                int seq, int normalize, float* out) {
    int cap = 0;
    size_t block = 0;   // the ids of a sub-batch; the mask and the token types follow them in in_dev
    return model_call(m, call, 0, [&] {
        MB_CHECK_ARG(ids && out, "NULL buffer");
        MB_CHECK_ARG(call == Call::TOKENS || normalize == 0 || normalize == 1,
                     "activation %d must be 0 (identity) or 1 (sigmoid)", normalize);
        check_tokens_args(m, n, seq);
        if (attn_mask && m->kind.text != TextKind::CLIP && m->kind.text != TextKind::COCA)
            check_prefix_mask(attn_mask, n, seq);
        cap = batch_cap_tokens(m, token_rows(m, seq));
        block = (size_t)std::min(n, cap) * seq;
        return block * 4 * (types ? 3 : 2);
    }, [&](Counter& c) {
        int32_t* d_ids = reinterpret_cast<int32_t*>(m->in_dev.get());
        int32_t* d_mask = d_ids + block;
        int32_t* d_types = types ? d_mask + block : nullptr;
        const size_t row_bytes = (size_t)seq * 4;
        host_batches(m, n, cap, [&](int o, int nb) {
            to_device(m, d_ids, ids + (size_t)o * seq, nb * row_bytes);
            if (attn_mask) to_device(m, d_mask, attn_mask + (size_t)o * seq, nb * row_bytes);
            if (types) to_device(m, d_types, types + (size_t)o * seq, nb * row_bytes);
        }, [&](int, int nb) {
            encode_tokens_dev(m, c, d_ids, attn_mask ? d_mask : nullptr, d_types, nb, seq, normalize, m->out_dev.get());
        }, {{out, m->out_dev.get(), (size_t)m->desc.embed_dim}});
    });
}

// The transformer tower b200_debug_layers runs: 0 vision, 1 text, if the model has one with layers.
const TowerW& layer_tower(b200_model* m, int tower) {
    MB_CHECK_ARG(tower == 0 || tower == 1, "tower %d must be 0 (vision) or 1 (text)", tower);
    const VisionKind vk = m->kind.vision;
    MB_CHECK_ARG(tower == 0 ? vk == VisionKind::CLIP_VIT || vk == VisionKind::SIGLIP_VIT || vk == VisionKind::EVA_VIT ||
                                  vk == VisionKind::COCA_VIT || vk == VisionKind::VIDEO_VIT
                            : m->kind.text != TextKind::NONE,
                 "this model has no transformer %s tower", tower == 0 ? "vision" : "text");
    return tower == 0 ? m->vision : m->text;
}

}  // namespace

extern "C" {

int b200_model_create(int device, const b200_model_desc* desc, b200_model** out) {
    return guarded([&] {
        MB_CHECK_ARG(desc && out, "NULL argument");
        *out = nullptr;
        require_sm90_device(device);
        MB_CHECK_ARG(desc->arch == B200_ARCH_CLIP || desc->arch == B200_ARCH_BERT || desc->arch == B200_ARCH_MPNET ||
                         desc->arch == B200_ARCH_SIGLIP || desc->arch == B200_ARCH_XLMR ||
                         desc->arch == B200_ARCH_CLIP_RESNET || desc->arch == B200_ARCH_CLIP_CONVNEXT ||
                         desc->arch == B200_ARCH_CLIP_EVA || desc->arch == B200_ARCH_GTE,
                     "unknown arch %d", desc->arch);
        MB_CHECK_ARG(desc->max_batch > 0, "max_batch must be positive");
        MB_CHECK_ARG(desc->embed_dim > 0 && desc->embed_dim <= 4096, "embed_dim out of range");
        const Kinds kind = resolve_kinds(*desc);
        MB_CHECK_ARG(kind.vision != VisionKind::NONE || kind.text != TextKind::NONE, "model has no tower");
        check_vision(*desc, kind.vision);
        check_text(*desc, kind);
        check_owl(*desc, kind);
        check_video(*desc, kind);
        DeviceGuard g(device);
        std::unique_ptr<b200_model> m(new b200_model());   // released under the guard if the set-up fails
        m->device = device;
        m->desc = *desc;
        m->sms = sm_count(device);
        m->own_stream = make_stream(cudaStreamNonBlocking);
        m->stream = m->own_stream.get();
        m->ev0 = make_event();
        m->ev1 = make_event();
        m->kind = kind;
        if (kind.vision == VisionKind::CLIP_VIT || kind.vision == VisionKind::SIGLIP_VIT ||
            kind.vision == VisionKind::EVA_VIT || kind.vision == VisionKind::COCA_VIT ||
            kind.vision == VisionKind::VIDEO_VIT)
            m->vision.d = desc->vision;
        if (kind.vision == VisionKind::RESNET) m->vision.d.image_size = desc->resnet_image_size;   // (no layers)
        if (kind.vision == VisionKind::CONVNEXT) {   // the stem, as a patch embedding (no layers)
            m->vision.d.image_size = desc->convnext_image_size;
            m->vision.d.patch = 4;
            m->vision.d.width = desc->convnext_dims[0];
        }
        if (kind.text != TextKind::NONE) m->text.d = desc->text;
        for (TowerW* T : {&m->vision, &m->text}) {
            if (T->d.heads > 0) T->aw = T->d.heads * kernel_head_dim(T->d.width / T->d.heads);
            T->mlp_h = T->d.mlp;
        }
        gemm::configure();
        *out = m.release();
    });
}

int b200_model_destroy(b200_model* m) {
    return guarded([&] {
        if (!m) return;
        DeviceGuard g(m->device);
        delete m;
    });
}

int b200_model_load_tensor(b200_model* m, const char* name, const float* data, int64_t numel) {
    return guarded([&] {
        MB_CHECK_ARG(m && name && data, "NULL argument");
        MB_CHECK_ARG(numel > 0, "numel must be positive");
        std::lock_guard<std::mutex> lk(m->mu);
        if (m->finalized) fail(B200_ERR_INVALID_ARG, "model is already finalized");
        DeviceGuard g(m->device);
        DeviceBuffer<float> b((size_t)numel);
        MB_CUDA(cudaMemcpy(b.get(), data, (size_t)numel * sizeof(float), cudaMemcpyHostToDevice));
        std::string key = name;
        // XLMRobertaModel checkpoints saved from a task head carry the encoder under "roberta."
        const bool xlmr = m->kind.text == TextKind::ROBERTA && !m->kind.mpnet;
        if (xlmr && key.compare(0, 8, "roberta.") == 0) key.erase(0, 8);
        // and NewModel checkpoints saved from a task head under "new."
        if (m->kind.text == TextKind::GTE && key.compare(0, 4, "new.") == 0) key.erase(0, 4);
        // and M-CLIP checkpoints (MultilingualCLIP) under "transformer.", beside their LinearTransformation
        if (m->desc.text_proj_dim > 0 && key.compare(0, 12, "transformer.") == 0) key.erase(0, 12);
        // and BertForSequenceClassification checkpoints under "bert.", beside their classifier
        if (m->kind.text == TextKind::BERT && key.compare(0, 5, "bert.") == 0) key.erase(0, 5);
        m->raw[key] = std::move(b);
    });
}

int b200_model_finalize(b200_model* m) {
    return guarded([&] {
        MB_CHECK_ARG(m != nullptr, "model is NULL");
        std::lock_guard<std::mutex> lk(m->mu);
        if (m->finalized) return;
        DeviceGuard g(m->device);
        build_vision(m);
        build_text(m);
        // workspaces for the towers' token rows, capped at ~24 GB of activations: larger calls are processed in
        // sub-batches
        const long long B = m->desc.max_batch, E = m->desc.embed_dim;
        long long max_tok = 0, max_w = 0, max_aw = 0, max_mlp = 0;
        for (const TowerW* T : {&m->vision, &m->text}) {
            if (T == &m->vision && m->kind.vision == VisionKind::CONVNEXT) continue;   // its own buffers (ConvnextW)
            max_tok = std::max(max_tok, B * std::max(1, T->frames) * T->tokens);   // (0 for a missing tower)
            max_w = std::max<long long>(max_w, T->d.width);
            max_aw = std::max<long long>({max_aw, T->d.width, T->aw});   // qkv and o: padded heads are wider
            max_mlp = std::max<long long>({max_mlp, fc1_cols(*T), T->map.mlp});
        }
        const long long bytes_per_tok = std::max<long long>(1, max_w * (4 + 2) + max_aw * (6 + 2) + max_mlp * 2);
        const long long cap_tok = (24LL << 30) / bytes_per_tok;
        m->max_tokens = std::min(max_tok, std::max<long long>(cap_tok, 1024));
        m->x = DeviceBuffer<float>((size_t)m->max_tokens * max_w);
        m->h = DeviceBuffer<__nv_bfloat16>((size_t)m->max_tokens * max_w);
        m->qkv = DeviceBuffer<__nv_bfloat16>((size_t)m->max_tokens * max_aw * 3);
        m->o = DeviceBuffer<__nv_bfloat16>((size_t)m->max_tokens * max_aw);
        m->u = DeviceBuffer<__nv_bfloat16>((size_t)m->max_tokens * max_mlp);
        if (m->kind.vision != VisionKind::NONE) {
            const int S = m->vision.d.image_size;
            m->resized = DeviceBuffer<uint8_t>((size_t)B * S * S * 3);
        }
        if (m->desc.owl_detect) m->det = DeviceBuffer<float>((size_t)B * m->vision.grid * m->vision.grid * 5);
        if (m->kind.vision == VisionKind::VIDEO_VIT) {
            const size_t S = m->vision.d.image_size;
            m->video_f32 = DeviceBuffer<float>((size_t)video_batch_cap(m) * m->vision.frames * 3 * S * S);
        }
        MB_CUDA(cudaStreamSynchronize(m->stream));
        m->aux = DeviceBuffer<int32_t>((size_t)B);
        m->out_dev = DeviceBuffer<float>((size_t)B * E);
        m->pooled = DeviceBuffer<float>((size_t)B * std::max(max_w, E));
        MB_CUDA(cudaStreamSynchronize(m->stream));
        m->finalized = true;
    });
}

int b200_model_encode_images_u8(b200_model* m, const uint8_t* hwc, int n, int h, int w, int normalize, float* out) {
    const size_t img_bytes = (size_t)h * w * 3;
    return model_call(m, Call::IMAGES, 0, [&] {
        check_u8_args(hwc && out, n, h, w);
        return (size_t)std::min(n, m->desc.max_batch) * img_bytes;
    }, [&](Counter& c) {
        host_batches(m, n, m->desc.max_batch, [&](int o, int nb) {
            to_device(m, m->in_dev.get(), hwc + (size_t)o * img_bytes, nb * img_bytes);
        }, [&](int, int nb) {
            encode_images_u8_dev(m, c, m->in_dev.get(), nb, h, w, normalize, m->out_dev.get());
        }, {{out, m->out_dev.get(), (size_t)m->desc.embed_dim}});
    });
}

int b200_model_encode_videos_u8(b200_model* m, const uint8_t* thwc, int n, int t, int h, int w, int normalize,
                                float* out) {
    const size_t video_bytes = (size_t)t * h * w * 3;
    return model_call(m, Call::VIDEOS, 0, [&] {
        check_u8_args(thwc && out, n, h, w);
        MB_CHECK_ARG(t == m->vision.frames, "videos of %d frames: the model takes %d", t, m->vision.frames);
        return (size_t)std::min(n, video_batch_cap(m)) * video_bytes;
    }, [&](Counter& c) {
        host_batches(m, n, video_batch_cap(m), [&](int o, int nb) {
            to_device(m, m->in_dev.get(), thwc + (size_t)o * video_bytes, nb * video_bytes);
        }, [&](int, int nb) {
            encode_videos_u8_dev(m, c, m->in_dev.get(), nb, h, w, normalize, m->out_dev.get());
        }, {{out, m->out_dev.get(), (size_t)m->desc.embed_dim}});
    });
}

int b200_model_encode_videos_u8_device(b200_model* m, const uint8_t* d_thwc, int n, int t, int h, int w, int normalize,
                                       float* d_out, int sync) {
    return model_call(m, Call::VIDEOS, sync, [&] {
        check_u8_args(d_thwc && d_out, n, h, w);
        MB_CHECK_ARG(t == m->vision.frames, "videos of %d frames: the model takes %d", t, m->vision.frames);
        return 0;
    }, [&](Counter& c) { encode_videos_u8_dev(m, c, d_thwc, n, h, w, normalize, d_out); });
}

int b200_model_detect_images_u8(b200_model* m, const uint8_t* hwc, int n, int h, int w, const int32_t* query_ids,
                                int seq, float* logits, float* boxes) {
    const size_t img_bytes = (size_t)h * w * 3;
    size_t ids_bytes = 0;   // in_dev holds the query's ids, then the images
    return model_call(m, Call::DETECT, 0, [&] {
        check_u8_args(hwc && query_ids && logits && boxes, n, h, w);
        MB_CHECK_ARG(seq > 0 && seq <= m->text.tokens, "query length %d out of range (1..%d)", seq, m->text.tokens);
        ids_bytes = round_up((size_t)seq * 4, 256);
        return ids_bytes + (size_t)std::min(n, image_batch_cap(m)) * img_bytes;
    }, [&](Counter& c) {
        const int P = m->vision.grid * m->vision.grid;
        const int32_t* d_ids = reinterpret_cast<const int32_t*>(m->in_dev.get());
        uint8_t* d_img = m->in_dev.get() + ids_bytes;
        float* d_logits = m->det.get();
        float* d_boxes = d_logits + (size_t)m->desc.max_batch * P;
        float* t = m->out_dev.get();   // the query's text embedding [embed_dim]
        to_device(m, m->in_dev.get(), query_ids, (size_t)seq * 4);
        forward_tokens(m, c, d_ids, nullptr, nullptr, 1, seq, 0, t);
        host_batches(m, n, image_batch_cap(m), [&](int o, int nb) {
            to_device(m, d_img, hwc + (size_t)o * img_bytes, nb * img_bytes);
        }, [&](int, int nb) {
            forward_detect(m, c, resize_images(m, c, d_img, nb, h, w), nb, t, d_logits, d_boxes);
        }, {{logits, d_logits, (size_t)P}, {boxes, d_boxes, (size_t)P * 4}});
    });
}

int b200_model_encode_images_u8_ragged(b200_model* m, const uint8_t* const* hwc, const int32_t* heights,
                                       const int32_t* widths, int n, int normalize, float* out) {
    auto bytes = [&](int i) { return (size_t)heights[i] * widths[i] * 3; };
    return model_call(m, Call::IMAGES, 0, [&] {
        MB_CHECK_ARG(out != nullptr, "NULL buffer");
        check_ragged_args(hwc, heights, widths, n);
        const int cap = image_batch_cap(m);
        size_t most = 0;   // the largest sub-batch's pixels: what in_dev must hold
        for (int o = 0; o < n; o += cap) {
            size_t sum = 0;
            for (int i = o; i < std::min(n, o + cap); ++i) sum += bytes(i);
            most = std::max(most, sum);
        }
        return most;
    }, [&](Counter& c) {
        std::vector<const uint8_t*> d_img((size_t)n);
        host_batches(m, n, image_batch_cap(m), [&](int o, int nb) {
            size_t off = 0;
            for (int i = o; i < o + nb;) {
                // one copy per run of images that lie back to back in host memory
                size_t run = bytes(i);
                d_img[i] = m->in_dev.get() + off;
                int j = i + 1;
                for (; j < o + nb && hwc[j] == hwc[j - 1] + bytes(j - 1); ++j) {
                    d_img[j] = d_img[i] + run;
                    run += bytes(j);
                }
                to_device(m, m->in_dev.get() + off, hwc[i], run);
                off += run;
                i = j;
            }
        }, [&](int o, int nb) {
            encode_images_u8_ragged_dev(m, c, d_img.data() + o, heights + o, widths + o, nb, normalize, m->out_dev.get());
        }, {{out, m->out_dev.get(), (size_t)m->desc.embed_dim}});
    });
}

int b200_model_encode_images_f32(b200_model* m, const float* chw, int n, int normalize, float* out) {
    size_t img = 0;   // floats per image
    return model_call(m, Call::IMAGES, 0, [&] {
        MB_CHECK_ARG(chw && out, "NULL buffer");
        MB_CHECK_ARG(n > 0, "n must be positive");
        img = (size_t)3 * m->vision.d.image_size * m->vision.d.image_size;
        return (size_t)std::min(n, image_batch_cap(m)) * img * 4;
    }, [&](Counter& c) {
        const float* d_chw = reinterpret_cast<const float*>(m->in_dev.get());
        host_batches(m, n, image_batch_cap(m), [&](int o, int nb) {
            to_device(m, m->in_dev.get(), chw + (size_t)o * img, nb * img * 4);
        }, [&](int, int nb) {
            forward_images(m, c, nullptr, d_chw, nb, normalize, m->out_dev.get());
        }, {{out, m->out_dev.get(), (size_t)m->desc.embed_dim}});
    });
}

int b200_model_encode_tokens(b200_model* m, const int32_t* ids, const int32_t* attn_mask, int n, int seq, int normalize,
                             float* out) {
    return tokens_host(m, Call::TOKENS, ids, attn_mask, nullptr, n, seq, normalize, out);
}

int b200_model_classify_tokens(b200_model* m, const int32_t* ids, const int32_t* attn_mask, const int32_t* type_ids,
                               int n, int seq, int activation, float* out) {
    return tokens_host(m, Call::CLASSIFY, ids, attn_mask, type_ids, n, seq, activation, out);
}

int b200_model_encode_images_u8_device(b200_model* m, const uint8_t* d_hwc, int n, int h, int w, int normalize,
                                       float* d_out, int sync) {
    return model_call(m, Call::IMAGES, sync, [&] {
        check_u8_args(d_hwc && d_out, n, h, w);
        return 0;
    }, [&](Counter& c) { encode_images_u8_dev(m, c, d_hwc, n, h, w, normalize, d_out); });
}

int b200_model_encode_images_u8_ragged_device(b200_model* m, const uint8_t* const* d_hwc, const int32_t* heights,
                                              const int32_t* widths, int n, int normalize, float* d_out, int sync) {
    return model_call(m, Call::IMAGES, sync, [&] {
        MB_CHECK_ARG(d_out != nullptr, "NULL buffer");
        check_ragged_args(d_hwc, heights, widths, n);
        return 0;
    }, [&](Counter& c) { encode_images_u8_ragged_dev(m, c, d_hwc, heights, widths, n, normalize, d_out); });
}

int b200_model_encode_tokens_device(b200_model* m, const int32_t* d_ids, const int32_t* d_attn_mask, int n, int seq,
                                    int normalize, float* d_out, int sync) {
    return model_call(m, Call::TOKENS, sync, [&] {
        MB_CHECK_ARG(d_ids && d_out, "NULL buffer");
        check_tokens_args(m, n, seq);
        return 0;
    }, [&](Counter& c) { encode_tokens_dev(m, c, d_ids, d_attn_mask, nullptr, n, seq, normalize, d_out); });
}

int b200_model_classify_tokens_device(b200_model* m, const int32_t* d_ids, const int32_t* d_attn_mask,
                                      const int32_t* d_type_ids, int n, int seq, int activation, float* d_out, int sync) {
    return model_call(m, Call::CLASSIFY, sync, [&] {
        MB_CHECK_ARG(d_ids && d_out, "NULL buffer");
        MB_CHECK_ARG(activation == 0 || activation == 1, "activation %d must be 0 (identity) or 1 (sigmoid)", activation);
        check_tokens_args(m, n, seq);
        return 0;
    }, [&](Counter& c) { encode_tokens_dev(m, c, d_ids, d_attn_mask, d_type_ids, n, seq, activation, d_out); });
}

int b200_model_set_stream(b200_model* m, void* cuda_stream, int use_external) {
    return guarded([&] {
        MB_CHECK_ARG(m != nullptr, "model is NULL");
        std::lock_guard<std::mutex> lk(m->mu);
        DeviceGuard g(m->device);
        MB_CUDA(cudaStreamSynchronize(m->stream));
        m->stream = use_external ? reinterpret_cast<cudaStream_t>(cuda_stream) : m->own_stream.get();
        m->external_stream = use_external != 0;   // a caller's stream may itself be under capture: no graphs there
    });
}

int b200_model_set_profiling(b200_model* m, int enable) {
    return guarded([&] {
        MB_CHECK_ARG(m != nullptr, "model is NULL");
        std::lock_guard<std::mutex> lk(m->mu);
        m->profiling = enable != 0;
        m->prof_n = 0;
    });
}

int b200_model_profile(b200_model* m, float* gemm_ms, int* gemm_launches, float* attention_ms, int* attention_launches) {
    return guarded([&] {
        MB_CHECK_ARG(m && gemm_ms && gemm_launches && attention_ms && attention_launches, "NULL argument");
        std::lock_guard<std::mutex> lk(m->mu);
        DeviceGuard g(m->device);
        float ms[2] = {0.f, 0.f};
        int cnt[2] = {0, 0};
        for (int i = 0; i < m->prof_n; ++i) {
            MB_CUDA(cudaEventSynchronize(m->prof_ev[2 * i + 1].get()));
            float t = 0.f;
            MB_CUDA(cudaEventElapsedTime(&t, m->prof_ev[2 * i].get(), m->prof_ev[2 * i + 1].get()));
            ms[m->prof_cls[i]] += t;
            ++cnt[m->prof_cls[i]];
        }
        *gemm_ms = ms[0];
        *gemm_launches = cnt[0];
        *attention_ms = ms[1];
        *attention_launches = cnt[1];
    });
}

int b200_debug_relative_position_buckets(int num_buckets, int max_distance, int max_len, int32_t* out) {
    return guarded([&] {
        MB_CHECK_ARG(out != nullptr, "NULL buffer");
        MB_CHECK_ARG(num_buckets >= 4 && num_buckets % 2 == 0 && max_distance > num_buckets / 4 && max_len > 0,
                     "bad bucket parameters");
        for (int d = -(max_len - 1); d <= max_len - 1; ++d)
            out[d + max_len - 1] = relative_position_bucket(d, num_buckets, max_distance);
    });
}

int b200_debug_layer_cols(b200_model* m, int tower, int32_t* out) {
    return guarded([&] {
        require_ready(m);
        MB_CHECK_ARG(out != nullptr, "NULL buffer");
        const TowerW& T = layer_tower(m, tower);
        out[0] = T.d.width;
        out[1] = T.aw;
        out[2] = fc1_cols(T);
    });
}

int b200_debug_layers(b200_model* m, int tower, int first, int count, const float* x_in, int B, int S,
                      const int32_t* kv_len, float* x_out, void* h_out, void* qkv_out, void* o_out, void* u_out,
                      void* stream) {
    return guarded([&] {
        require_ready(m);
        MB_CHECK_ARG(x_in != nullptr, "NULL buffer");
        std::lock_guard<std::mutex> lk(m->mu);
        const TowerW& T = layer_tower(m, tower);
        const bool vision = tower == 0;
        const TextKind tk = m->kind.text;
        const int L = (int)T.layers.size();
        MB_CHECK_ARG(first >= 0 && count > 0 && first <= L - count, "layers [%d, %d + %d) outside the tower's %d", first,
                     first, count, L);
        const int per = vision ? std::max(1, T.frames) : 1;   // a video tower's sequences are its videos' frames
        MB_CHECK_ARG(B > 0 && B % per == 0 && B / per <= m->desc.max_batch, "B %d out of range (1..%d%s)", B,
                     m->desc.max_batch * per, per > 1 ? ", a multiple of the frames" : "");
        MB_CHECK_ARG(vision ? S == T.tokens : S > 0 && S <= T.tokens, "S %d: the %s tower takes %s%d tokens", S,
                     vision ? "vision" : "text", vision ? "" : "1..", T.tokens);
        MB_CHECK_ARG((long long)B * S <= m->max_tokens, "B * S = %lld rows exceed the workspace's %lld",
                     (long long)B * S, m->max_tokens);
        // the mask of the tower's forward pass (forward_vit, forward_tokens_eager)
        const int mask = vision || tk == TextKind::SIGLIP                 ? attention::MASK_NONE
                         : tk == TextKind::CLIP || tk == TextKind::COCA ? attention::MASK_CAUSAL
                                                                        : attention::MASK_KEYLEN;
        DeviceGuard g(m->device);
        // an encode call with sync = 0 may still be using the workspaces on the model's stream
        MB_CUDA(cudaStreamSynchronize(m->stream));
        const cudaStream_t s = static_cast<cudaStream_t>(stream);
        std::vector<int32_t> lens((size_t)B, S);
        if (mask == attention::MASK_KEYLEN && kv_len) {
            MB_CUDA(cudaMemcpyAsync(lens.data(), kv_len, lens.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
            MB_CUDA(cudaStreamSynchronize(s));
            for (int b = 0; b < B; ++b)
                MB_CHECK_ARG(lens[b] >= 0 && lens[b] <= S, "kv_len[%d] = %d outside 0..%d", b, lens[b], S);
        }
        const cudaStream_t saved = m->stream;
        m->stream = s;
        try {
            const size_t M = (size_t)B * S, w = T.d.width;
            MB_CUDA(cudaMemcpyAsync(m->x.get(), x_in, M * w * sizeof(float), cudaMemcpyDeviceToDevice, s));
            // a post-LN tower's layers start from the embedding LayerNorm's two outputs, x and h = bf16(x)
            if (!T.pre_ln) kernels::f32_to_bf16(m->x.get(), m->h.get(), (long long)(M * w), s);
            if (mask == attention::MASK_KEYLEN) {
                MB_CUDA(cudaMemcpyAsync(m->aux.get(), lens.data(), lens.size() * sizeof(int32_t), cudaMemcpyHostToDevice,
                                        s));
                MB_CUDA(cudaStreamSynchronize(s));   // `lens` is pageable
            }
            Counter c;
            run_layers(m, c, T, B, S, mask, first, count);
            const size_t aw = T.aw, fc1 = fc1_cols(T);
            if (x_out) MB_CUDA(cudaMemcpyAsync(x_out, m->x.get(), M * w * sizeof(float), cudaMemcpyDeviceToDevice, s));
            if (h_out) MB_CUDA(cudaMemcpyAsync(h_out, m->h.get(), M * w * 2, cudaMemcpyDeviceToDevice, s));
            if (qkv_out) MB_CUDA(cudaMemcpyAsync(qkv_out, m->qkv.get(), M * 3 * aw * 2, cudaMemcpyDeviceToDevice, s));
            if (o_out) MB_CUDA(cudaMemcpyAsync(o_out, m->o.get(), M * aw * 2, cudaMemcpyDeviceToDevice, s));
            if (u_out) MB_CUDA(cudaMemcpyAsync(u_out, m->u.get(), M * fc1 * 2, cudaMemcpyDeviceToDevice, s));
            MB_CUDA(cudaStreamSynchronize(s));
        } catch (...) {
            m->stream = saved;
            throw;
        }
        m->stream = saved;
    });
}

int b200_model_last_timing(b200_model* m, float* ms, int* launches) {
    return guarded([&] {
        MB_CHECK_ARG(m && ms && launches, "NULL argument");
        std::lock_guard<std::mutex> lk(m->mu);
        DeviceGuard g(m->device);
        if (!m->timing_valid) fail(B200_ERR_INVALID_ARG, "no encode call has been timed yet");
        MB_CUDA(cudaEventSynchronize(m->ev1.get()));
        MB_CUDA(cudaEventElapsedTime(ms, m->ev0.get(), m->ev1.get()));
        *launches = m->last_launches;
    });
}

}  // extern "C"
