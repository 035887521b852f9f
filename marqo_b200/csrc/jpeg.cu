// Baseline JPEG decode for the ingest path (SURVEY §8 f4): the reference decodes every image with Pillow on a download
// thread (`Image.open(...)` in src/marqo/core/inference/image_download.py:146-152, pixels materialised by the transform
// at src/marqo/tensor_search/add_docs.py:129-134).  Pillow wraps libjpeg-turbo; its default decode path is
//     Huffman decode -> dequantise + "islow" integer IDCT (jidctint.c) -> fancy (triangle) chroma upsampling
//     (jdsample.c h2v1 / h2v2) -> fixed-point YCbCr -> RGB (jdcolor.c),
// every stage integer arithmetic, so a re-implementation can be BIT-EXACT — and this one is tested to be
// (tests/test_jpeg.py compares against Pillow pixel for pixel).
//
// Split: the entropy-coded segment is inherently serial per image -> decoded on the host (one image per thread, images
// of a batch in parallel) into int16 coefficient blocks; everything after it is per-block / per-pixel -> two CUDA
// kernels over the whole batch:
//     idct_kernel        one thread per 8x8 block: dequantise, islow IDCT, +128, clamp -> uint8 component planes
//     upsample_rgb_kernel one thread per output pixel: fancy upsampling of Cb / Cr at that pixel, YCbCr -> RGB -> HWC
// The arithmetic lives in __host__ __device__ functions shared with a host reference (b200_debug_jpeg_decode_host) that
// the CPU test suite checks against Pillow, so the kernels are verified even where no GPU exists.
//
// Supported: baseline / extended-sequential Huffman JPEG (SOF0 / SOF1), 8-bit, 1 component (grey) or 3 components
// (YCbCr) with luma sampling 1x1, 2x1 or 2x2 and 1x1 chroma, restart intervals, interleaved single scan.  Everything else
// (progressive, arithmetic coding, CMYK / YCCK, RGB-tagged, 12-bit, exotic sampling) returns B200_ERR_UNSUPPORTED per
// image and the adapter falls back to Pillow for that image.
#include <algorithm>
#include <atomic>
#include <cstring>
#include <memory>
#include <thread>
#include <vector>

#include "common.cuh"

namespace mb {
namespace jpeg {

// ---------------------------------------------------------------------------------------------- shared arithmetic
#define JF __host__ __device__ __forceinline__

JF int clamp_u8(int x) { return x < 0 ? 0 : (x > 255 ? 255 : x); }
JF int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }   // arithmetic shift, as libjpeg's DESCALE

// jidctint.c jpeg_idct_islow (8x8): CONST_BITS = 13, PASS1_BITS = 2.  `coef` are the quantised coefficients in natural
// (row-major) order, `q` the quantisation table in natural order; `out` receives 64 samples (row-major).
JF void idct_islow(const int16_t* coef, const uint16_t* q, uint8_t* out, int out_stride) {
    constexpr int CB = 13, P1 = 2;
    constexpr int F_0_298631336 = 2446, F_0_390180644 = 3196, F_0_541196100 = 4433, F_0_765366865 = 6270,
                  F_0_899976223 = 7373, F_1_175875602 = 9633, F_1_501321110 = 12299, F_1_847759065 = 15137,
                  F_1_961570560 = 16069, F_2_053119869 = 16819, F_2_562915447 = 20995, F_3_072711026 = 25172;
    int ws[64];
    for (int c = 0; c < 8; ++c) {   // pass 1: columns
        const int i0 = coef[c] * q[c], i1 = coef[8 + c] * q[8 + c], i2 = coef[16 + c] * q[16 + c],
                  i3 = coef[24 + c] * q[24 + c], i4 = coef[32 + c] * q[32 + c], i5 = coef[40 + c] * q[40 + c],
                  i6 = coef[48 + c] * q[48 + c], i7 = coef[56 + c] * q[56 + c];
        int z2 = i2, z3 = i6;
        int z1 = (z2 + z3) * F_0_541196100;
        int tmp2 = z1 + z3 * (-F_1_847759065);
        int tmp3 = z1 + z2 * F_0_765366865;
        z2 = i0;
        z3 = i4;
        int tmp0 = (z2 + z3) * (1 << CB);
        int tmp1 = (z2 - z3) * (1 << CB);
        const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
        tmp0 = i7;
        tmp1 = i5;
        tmp2 = i3;
        tmp3 = i1;
        z1 = tmp0 + tmp3;
        z2 = tmp1 + tmp2;
        z3 = tmp0 + tmp2;
        int z4 = tmp1 + tmp3;
        const int z5 = (z3 + z4) * F_1_175875602;
        tmp0 *= F_0_298631336;
        tmp1 *= F_2_053119869;
        tmp2 *= F_3_072711026;
        tmp3 *= F_1_501321110;
        z1 *= -F_0_899976223;
        z2 *= -F_2_562915447;
        z3 *= -F_1_961570560;
        z4 *= -F_0_390180644;
        z3 += z5;
        z4 += z5;
        tmp0 += z1 + z3;
        tmp1 += z2 + z4;
        tmp2 += z2 + z3;
        tmp3 += z1 + z4;
        ws[c] = descale(tmp10 + tmp3, CB - P1);
        ws[56 + c] = descale(tmp10 - tmp3, CB - P1);
        ws[8 + c] = descale(tmp11 + tmp2, CB - P1);
        ws[48 + c] = descale(tmp11 - tmp2, CB - P1);
        ws[16 + c] = descale(tmp12 + tmp1, CB - P1);
        ws[40 + c] = descale(tmp12 - tmp1, CB - P1);
        ws[24 + c] = descale(tmp13 + tmp0, CB - P1);
        ws[32 + c] = descale(tmp13 - tmp0, CB - P1);
    }
    for (int r = 0; r < 8; ++r) {   // pass 2: rows
        const int* w = ws + 8 * r;
        int z2 = w[2], z3 = w[6];
        int z1 = (z2 + z3) * F_0_541196100;
        int tmp2 = z1 + z3 * (-F_1_847759065);
        int tmp3 = z1 + z2 * F_0_765366865;
        int tmp0 = (w[0] + w[4]) * (1 << CB);
        int tmp1 = (w[0] - w[4]) * (1 << CB);
        const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
        tmp0 = w[7];
        tmp1 = w[5];
        tmp2 = w[3];
        tmp3 = w[1];
        z1 = tmp0 + tmp3;
        z2 = tmp1 + tmp2;
        z3 = tmp0 + tmp2;
        int z4 = tmp1 + tmp3;
        const int z5 = (z3 + z4) * F_1_175875602;
        tmp0 *= F_0_298631336;
        tmp1 *= F_2_053119869;
        tmp2 *= F_3_072711026;
        tmp3 *= F_1_501321110;
        z1 *= -F_0_899976223;
        z2 *= -F_2_562915447;
        z3 *= -F_1_961570560;
        z4 *= -F_0_390180644;
        z3 += z5;
        z4 += z5;
        tmp0 += z1 + z3;
        tmp1 += z2 + z4;
        tmp2 += z2 + z3;
        tmp3 += z1 + z4;
        uint8_t* o = out + (size_t)r * out_stride;
        constexpr int SH = CB + P1 + 3;
        o[0] = (uint8_t)clamp_u8(descale(tmp10 + tmp3, SH) + 128);
        o[7] = (uint8_t)clamp_u8(descale(tmp10 - tmp3, SH) + 128);
        o[1] = (uint8_t)clamp_u8(descale(tmp11 + tmp2, SH) + 128);
        o[6] = (uint8_t)clamp_u8(descale(tmp11 - tmp2, SH) + 128);
        o[2] = (uint8_t)clamp_u8(descale(tmp12 + tmp1, SH) + 128);
        o[5] = (uint8_t)clamp_u8(descale(tmp12 - tmp1, SH) + 128);
        o[3] = (uint8_t)clamp_u8(descale(tmp13 + tmp0, SH) + 128);
        o[4] = (uint8_t)clamp_u8(descale(tmp13 - tmp0, SH) + 128);
    }
}

// One image's geometry, shared by host and device.
struct ImageDesc {
    int width, height;       // output size
    int ncomp;               // 1 or 3
    int hs, vs;              // luma sampling factors (chroma is 1x1): 1x1, 2x1 or 2x2
    int comp_w[3], comp_h[3];          // TRUE downsampled component size (jpeg_component_info.downsampled_*)
    int plane_w[3], plane_h[3];        // padded to whole blocks (what the IDCT writes)
    int blocks_w[3], blocks_h[3];      // blocks per row / column in the plane
    long long coef_off[3];   // first coefficient block of the component in the batch's coefficient buffer (in blocks)
    long long plane_off[3];  // first byte of the component plane in the batch's plane buffer
    long long block_base;    // number of blocks of all previous images (idct grid mapping)
    long long pixel_base;    // number of output pixels of all previous images (upsample grid mapping)
    int qtab[3];             // quantisation table index per component
    uint16_t q[4][64];       // natural order
    uint8_t* out;            // device (or host) HWC RGB destination
};

// jdsample.c: the upsampled chroma sample at output position (x, y) of a plane `p` (true size cw x ch, row pitch pw).
//   1x1: the sample itself.
//   h2v1_fancy_upsample: 3/4 nearer + 1/4 further column, rounding 1 (even outputs) / 2 (odd outputs); the first and the
//     last output column copy their input sample.
//   Components of true width <= 2 are replicated instead (libjpeg only installs the fancy routines for wider ones).
//   h2v2_fancy_upsample: column sums 3 * nearer row + further row, then (3 * this + neighbour + 8 or 7) >> 4; edge
//     columns (this * 4 + 8 or 7) >> 4.  Rows above the first / below the last TRUE row replicate that row
//     (jdmainct.c context rows: set_wraparound_pointers / set_bottom_pointers).
JF int upsampled(const uint8_t* p, int pw, int cw, int ch, int hs, int vs, int x, int y) {
    if (hs == 1 && vs == 1) return p[(size_t)y * pw + x];
    const int i = x >> 1;
    // jinit_upsampler: fancy upsampling only when downsampled_width > 2; narrower components are replicated
    // (h2v1_upsample / h2v2_upsample)
    if (cw <= 2) return p[(size_t)(vs == 2 ? (y >> 1) : y) * pw + i];
    if (vs == 1) {   // h2v1
        const uint8_t* row = p + (size_t)y * pw;
        const int v = row[i];
        if ((x & 1) == 0) return i == 0 ? v : (3 * v + row[i - 1] + 1) >> 2;
        return i == cw - 1 ? v : (3 * v + row[i + 1] + 2) >> 2;
    }
    // h2v2
    const int j = y >> 1;
    const int jn = (y & 1) ? min(j + 1, ch - 1) : max(j - 1, 0);   // further row: below for odd, above for even outputs
    const uint8_t* r0 = p + (size_t)j * pw;
    const uint8_t* r1 = p + (size_t)jn * pw;
    const int cur = 3 * r0[i] + r1[i];
    if ((x & 1) == 0) {
        if (i == 0) return (cur * 4 + 8) >> 4;
        return (cur * 3 + (3 * r0[i - 1] + r1[i - 1]) + 8) >> 4;
    }
    if (i == cw - 1) return (cur * 4 + 7) >> 4;
    return (cur * 3 + (3 * r0[i + 1] + r1[i + 1]) + 7) >> 4;
}

// jdcolor.c build_ycc_rgb_table / ycc_rgb_convert: SCALEBITS = 16, FIX(x) = (int)(x * 65536 + 0.5).
JF void ycc_to_rgb(int y, int cb, int cr, uint8_t* rgb) {
    constexpr int ONE_HALF = 1 << 15;
    const int xb = cb - 128, xr = cr - 128;
    const int cr_r = (91881 * xr + ONE_HALF) >> 16;           // FIX(1.40200)
    const int cb_b = (116130 * xb + ONE_HALF) >> 16;          // FIX(1.77200)
    const int g = (-22554 * xb + ONE_HALF + -46802 * xr) >> 16;   // Cb_g_tab (with ONE_HALF) + Cr_g_tab
    rgb[0] = (uint8_t)clamp_u8(y + cr_r);
    rgb[1] = (uint8_t)clamp_u8(y + g);
    rgb[2] = (uint8_t)clamp_u8(y + cb_b);
}

JF void output_pixel(const ImageDesc& d, const uint8_t* planes, int x, int y) {
    uint8_t* o = d.out + ((size_t)y * d.width + x) * 3;
    const int Y = planes[d.plane_off[0] + (size_t)y * d.plane_w[0] + x];
    if (d.ncomp == 1) {
        o[0] = o[1] = o[2] = (uint8_t)Y;   // Pillow: mode "L" -> convert("RGB") replicates
        return;
    }
    const int cb = upsampled(planes + d.plane_off[1], d.plane_w[1], d.comp_w[1], d.comp_h[1], d.hs, d.vs, x, y);
    const int cr = upsampled(planes + d.plane_off[2], d.plane_w[2], d.comp_w[2], d.comp_h[2], d.hs, d.vs, x, y);
    ycc_to_rgb(Y, cb, cr, o);
}

// ---------------------------------------------------------------------------------------------- kernels
__global__ void idct_kernel(const ImageDesc* __restrict__ descs, int n_images, const int16_t* __restrict__ coefs,
                            uint8_t* __restrict__ planes, long long total_blocks) {
    const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= total_blocks) return;
    int lo = 0, hi = n_images - 1;   // image owning block b: last image with block_base <= b
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (descs[mid].block_base <= b) lo = mid;
        else hi = mid - 1;
    }
    const ImageDesc& d = descs[lo];
    long long local = b - d.block_base;
    int c = 0;
    for (; c < d.ncomp - 1; ++c) {
        const long long nb = (long long)d.blocks_w[c] * d.blocks_h[c];
        if (local < nb) break;
        local -= nb;
    }
    const int by = (int)(local / d.blocks_w[c]), bx = (int)(local % d.blocks_w[c]);
    idct_islow(coefs + (d.coef_off[c] + local) * 64, d.q[d.qtab[c]],
               planes + d.plane_off[c] + ((size_t)by * 8) * d.plane_w[c] + bx * 8, d.plane_w[c]);
}

__global__ void upsample_rgb_kernel(const ImageDesc* __restrict__ descs, int n_images, const uint8_t* __restrict__ planes,
                                    long long total_pixels) {
    const long long px = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (px >= total_pixels) return;
    int lo = 0, hi = n_images - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (descs[mid].pixel_base <= px) lo = mid;
        else hi = mid - 1;
    }
    const ImageDesc& d = descs[lo];
    const long long local = px - d.pixel_base;
    output_pixel(d, planes, (int)(local % d.width), (int)(local / d.width));
}

// ---------------------------------------------------------------------------------------------- host: parse + Huffman
struct Unsupported {
    const char* why;
};

static const uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

struct HuffTable {
    bool present = false;
    uint8_t bits[17] = {0};
    uint8_t vals[256] = {0};
    // canonical decoding: for code length l, codes [mincode[l], maxcode[l]] map to vals[valptr[l] + code - mincode[l]]
    int mincode[17], maxcode[18], valptr[17];
    uint8_t look_len[512];   // 9-bit lookahead: code length (0 = longer than 9 bits)
    uint8_t look_sym[512];
    void build() {
        int code = 0, k = 0;
        for (int l = 1; l <= 16; ++l) {
            valptr[l] = k;
            mincode[l] = code;
            code += bits[l];
            k += bits[l];
            maxcode[l] = bits[l] ? code - 1 : -1;
            code <<= 1;
        }
        maxcode[17] = 0x7fffffff;
        memset(look_len, 0, sizeof(look_len));
        int c = 0, p = 0;
        for (int l = 1; l <= 9; ++l) {
            for (int i = 0; i < bits[l]; ++i, ++p, ++c) {
                const int first = c << (9 - l);
                for (int f = 0; f < (1 << (9 - l)); ++f) {
                    look_len[first + f] = (uint8_t)l;
                    look_sym[first + f] = vals[p];
                }
            }
            c <<= 1;
        }
    }
};

struct BitReader {
    const uint8_t* p;
    const uint8_t* end;
    uint64_t acc = 0;
    int nbits = 0;
    bool hit_marker = false;
    void fill() {
        while (nbits <= 56) {
            int byte = 0;
            if (!hit_marker && p < end) {
                byte = *p;
                if (byte == 0xFF) {
                    if (p + 1 < end && p[1] == 0x00) {
                        p += 2;
                    } else {   // a marker (RSTn / EOI): feed zeros until the caller resynchronises
                        hit_marker = true;
                        byte = 0;
                    }
                } else {
                    ++p;
                }
            }
            acc |= (uint64_t)byte << (56 - nbits);
            nbits += 8;
        }
    }
    inline int peek(int n) { return (int)(acc >> (64 - n)); }
    inline void skip(int n) {
        acc <<= n;
        nbits -= n;
    }
    inline int get(int n) {
        if (n == 0) return 0;
        const int v = peek(n);
        skip(n);
        return v;
    }
    void reset_at(const uint8_t* np) {
        p = np;
        acc = 0;
        nbits = 0;
        hit_marker = false;
    }
};

static inline int huff_decode(BitReader& br, const HuffTable& h) {
    if (br.nbits < 16) br.fill();
    const int look = br.peek(9);
    const int l = h.look_len[look];
    if (l) {
        br.skip(l);
        return h.look_sym[look];
    }
    int code = br.peek(10), len = 10;
    while (len <= 16 && code > h.maxcode[len]) {
        ++len;
        code = br.peek(len);
    }
    if (len > 16) throw Unsupported{"corrupt Huffman code"};
    br.skip(len);
    return h.vals[h.valptr[len] + code - h.mincode[len]];
}

static inline int extend(int v, int s) { return v < (1 << (s - 1)) ? v - (1 << s) + 1 : v; }

struct Parsed {
    ImageDesc d;
    std::vector<int16_t> coefs;   // all components, blocks in plane raster order
};

static inline int be16(const uint8_t* p) { return (p[0] << 8) | p[1]; }

// Parses the headers and entropy-decodes the scan.  Throws Unsupported for anything outside the supported subset.
static void parse_and_decode(const uint8_t* data, size_t n, Parsed& out) {
    if (n < 4 || data[0] != 0xFF || data[1] != 0xD8) throw Unsupported{"not a JPEG file"};
    HuffTable dc[4], ac[4];
    ImageDesc& d = out.d;
    memset(&d, 0, sizeof(d));
    int comp_id[3] = {0}, comp_h[3] = {0}, comp_v[3] = {0};
    int restart_interval = 0;
    bool have_sof = false;
    int adobe_transform = -1;
    size_t pos = 2;
    while (true) {
        while (pos < n && data[pos] != 0xFF) ++pos;   // tolerate garbage between segments like libjpeg's next_marker
        while (pos < n && data[pos] == 0xFF) ++pos;
        if (pos >= n) throw Unsupported{"truncated JPEG (no scan)"};
        const int marker = data[pos++];
        if (marker == 0xD8 || (marker >= 0xD0 && marker <= 0xD7) || marker == 0x01) continue;
        if (marker == 0xD9) throw Unsupported{"JPEG without a scan"};
        if (pos + 2 > n) throw Unsupported{"truncated JPEG"};
        const int len = be16(data + pos);
        if (len < 2 || pos + len > n) throw Unsupported{"truncated JPEG segment"};
        const uint8_t* seg = data + pos + 2;
        const int slen = len - 2;
        if (marker == 0xDB) {   // DQT
            int o = 0;
            while (o < slen) {
                const int pq = seg[o] >> 4, tq = seg[o] & 15;
                ++o;
                if (tq > 3) throw Unsupported{"bad quantisation table id"};
                if (pq != 0) throw Unsupported{"16-bit quantisation tables"};
                if (o + 64 > slen) throw Unsupported{"truncated DQT"};
                for (int i = 0; i < 64; ++i) d.q[tq][kZigzag[i]] = seg[o + i];
                o += 64;
            }
        } else if (marker == 0xC4) {   // DHT
            int o = 0;
            while (o < slen) {
                const int tc = seg[o] >> 4, th = seg[o] & 15;
                ++o;
                if (tc > 1 || th > 3 || o + 16 > slen) throw Unsupported{"bad Huffman table"};
                HuffTable& h = tc ? ac[th] : dc[th];
                int total = 0;
                h.bits[0] = 0;
                for (int i = 1; i <= 16; ++i) {
                    h.bits[i] = seg[o + i - 1];
                    total += h.bits[i];
                }
                o += 16;
                if (total > 256 || o + total > slen) throw Unsupported{"bad Huffman table"};
                memcpy(h.vals, seg + o, total);
                o += total;
                h.present = true;
                h.build();
            }
        } else if (marker == 0xC0 || marker == 0xC1) {   // SOF0 / SOF1
            if (slen < 6) throw Unsupported{"truncated SOF"};
            if (seg[0] != 8) throw Unsupported{"sample precision other than 8 bits"};
            d.height = be16(seg + 1);
            d.width = be16(seg + 3);
            d.ncomp = seg[5];
            if (d.height <= 0 || d.width <= 0) throw Unsupported{"empty image"};
            if (d.ncomp != 1 && d.ncomp != 3) throw Unsupported{"component count other than 1 or 3 (CMYK / YCCK)"};
            if (slen < 6 + 3 * d.ncomp) throw Unsupported{"truncated SOF"};
            for (int c = 0; c < d.ncomp; ++c) {
                comp_id[c] = seg[6 + 3 * c];
                comp_h[c] = seg[7 + 3 * c] >> 4;
                comp_v[c] = seg[7 + 3 * c] & 15;
                d.qtab[c] = seg[8 + 3 * c];
                if (d.qtab[c] > 3) throw Unsupported{"bad quantisation table id"};
            }
            have_sof = true;
        } else if (marker == 0xC2 || (marker >= 0xC3 && marker <= 0xCF && marker != 0xC4 && marker != 0xC8 && marker != 0xCC)) {
            throw Unsupported{"progressive / lossless / arithmetic-coded JPEG"};
        } else if (marker == 0xCC) {
            throw Unsupported{"arithmetic-coded JPEG"};
        } else if (marker == 0xDD) {   // DRI
            if (slen < 2) throw Unsupported{"truncated DRI"};
            restart_interval = be16(seg);
        } else if (marker == 0xEE) {   // APP14 Adobe
            if (slen >= 12 && memcmp(seg, "Adobe", 5) == 0) adobe_transform = seg[11];
        } else if (marker == 0xDA) {   // SOS
            if (!have_sof) throw Unsupported{"scan before frame header"};
            if (slen < 1 || seg[0] != d.ncomp) throw Unsupported{"non-interleaved scans"};
            if (slen < 1 + 2 * d.ncomp + 3) throw Unsupported{"truncated SOS"};
            int td[3], ta[3];
            for (int c = 0; c < d.ncomp; ++c) {
                if (seg[1 + 2 * c] != comp_id[c]) throw Unsupported{"scan component order differs from the frame"};
                td[c] = seg[2 + 2 * c] >> 4;
                ta[c] = seg[2 + 2 * c] & 15;
                if (td[c] > 3 || ta[c] > 3 || !dc[td[c]].present || !ac[ta[c]].present)
                    throw Unsupported{"scan refers to a missing Huffman table"};
            }
            // colour space as libjpeg guesses it (jdapimin.c default_decompress_parms)
            if (d.ncomp == 3) {
                if (adobe_transform == 0) throw Unsupported{"Adobe RGB-tagged JPEG"};
                if (adobe_transform < 0 && comp_id[0] == 'R' && comp_id[1] == 'G' && comp_id[2] == 'B')
                    throw Unsupported{"RGB-tagged JPEG"};
                if (comp_h[1] != 1 || comp_v[1] != 1 || comp_h[2] != 1 || comp_v[2] != 1)
                    throw Unsupported{"chroma sampling factors other than 1x1"};
                d.hs = comp_h[0];
                d.vs = comp_v[0];
                if (!((d.hs == 1 && d.vs == 1) || (d.hs == 2 && d.vs == 1) || (d.hs == 2 && d.vs == 2)))
                    throw Unsupported{"luma sampling other than 1x1, 2x1, 2x2"};
            } else {
                d.hs = d.vs = 1;   // a single component is never interleaved: its own sampling factors do not matter
                comp_h[0] = comp_v[0] = 1;
            }
            const int mcu_w = 8 * d.hs, mcu_h = 8 * d.vs;
            const int mcus_x = (d.width + mcu_w - 1) / mcu_w, mcus_y = (d.height + mcu_h - 1) / mcu_h;
            long long blocks = 0;
            for (int c = 0; c < d.ncomp; ++c) {
                const int h = c == 0 ? d.hs : 1, v = c == 0 ? d.vs : 1;
                d.blocks_w[c] = mcus_x * h;
                d.blocks_h[c] = mcus_y * v;
                d.plane_w[c] = d.blocks_w[c] * 8;
                d.plane_h[c] = d.blocks_h[c] * 8;
                d.comp_w[c] = (d.width * h + d.hs - 1) / d.hs;     // ceil(width * h_samp / max_h_samp)
                d.comp_h[c] = (d.height * v + d.vs - 1) / d.vs;
                d.coef_off[c] = blocks;
                blocks += (long long)d.blocks_w[c] * d.blocks_h[c];
            }
            if (blocks > (1ll << 24)) throw Unsupported{"image too large"};
            out.coefs.assign((size_t)blocks * 64, 0);
            // ---- entropy-coded segment
            BitReader br;
            br.reset_at(seg + slen);
            br.end = data + n;
            int pred[3] = {0, 0, 0};
            int until_restart = restart_interval;
            int next_rst = 0;
            for (int my = 0; my < mcus_y; ++my) {
                for (int mx = 0; mx < mcus_x; ++mx) {
                    if (restart_interval && until_restart == 0) {
                        // byte-align, expect RSTn
                        const uint8_t* q = br.p;
                        while (q + 1 < br.end && !(q[0] == 0xFF && q[1] >= 0xD0 && q[1] <= 0xD7)) ++q;
                        if (q + 1 >= br.end || q[1] != 0xD0 + next_rst) throw Unsupported{"missing restart marker"};
                        br.reset_at(q + 2);
                        next_rst = (next_rst + 1) & 7;
                        pred[0] = pred[1] = pred[2] = 0;
                        until_restart = restart_interval;
                    }
                    for (int c = 0; c < d.ncomp; ++c) {
                        const int h = c == 0 ? d.hs : 1, v = c == 0 ? d.vs : 1;
                        for (int vy = 0; vy < v; ++vy) {
                            for (int hx = 0; hx < h; ++hx) {
                                const int bx = mx * h + hx, by = my * v + vy;
                                int16_t* blk = out.coefs.data() + ((size_t)d.coef_off[c] + (size_t)by * d.blocks_w[c] + bx) * 64;
                                int s = huff_decode(br, dc[td[c]]);
                                if (s > 11) throw Unsupported{"corrupt DC coefficient"};
                                int diff = 0;
                                if (s) {
                                    if (br.nbits < s) br.fill();
                                    diff = extend(br.get(s), s);
                                }
                                pred[c] += diff;
                                blk[0] = (int16_t)pred[c];
                                for (int k = 1; k < 64;) {
                                    const int rs = huff_decode(br, ac[ta[c]]);
                                    const int r = rs >> 4;
                                    s = rs & 15;
                                    if (s == 0) {
                                        if (r != 15) break;   // EOB
                                        k += 16;              // ZRL
                                        continue;
                                    }
                                    k += r;
                                    if (k > 63) throw Unsupported{"corrupt AC run"};
                                    if (br.nbits < s) br.fill();
                                    blk[kZigzag[k]] = (int16_t)extend(br.get(s), s);
                                    ++k;
                                }
                            }
                        }
                    }
                    if (restart_interval) --until_restart;
                }
            }
            return;
        }
        pos += len;
    }
}

static void layout_batch(std::vector<Parsed>& imgs, const std::vector<int>& ok, std::vector<ImageDesc>& descs,
                         long long& total_blocks, long long& total_pixels, long long& plane_bytes) {
    total_blocks = total_pixels = plane_bytes = 0;
    for (int i : ok) {
        ImageDesc d = imgs[i].d;
        d.block_base = total_blocks;
        d.pixel_base = total_pixels;
        long long nb = 0;
        for (int c = 0; c < d.ncomp; ++c) {
            d.coef_off[c] += total_blocks;
            d.plane_off[c] = plane_bytes;
            plane_bytes += (long long)d.plane_w[c] * d.plane_h[c];
            nb += (long long)d.blocks_w[c] * d.blocks_h[c];
        }
        total_blocks += nb;
        total_pixels += (long long)d.width * d.height;
        descs.push_back(d);
    }
}

static void decode_parallel(const uint8_t* const* files, const size_t* nbytes, int n, std::vector<Parsed>& imgs,
                            int32_t* status, std::vector<std::string>& why) {
    std::atomic<int> next{0};
    auto work = [&] {
        for (int i = next.fetch_add(1); i < n; i = next.fetch_add(1)) {
            try {
                if (!files[i]) throw Unsupported{"NULL file"};
                parse_and_decode(files[i], nbytes[i], imgs[i]);
                status[i] = B200_OK;
            } catch (const Unsupported& u) {
                status[i] = B200_ERR_UNSUPPORTED;
                why[i] = u.why;
            } catch (const std::bad_alloc&) {
                status[i] = B200_ERR_OOM;
            }
        }
    };
    const int nt = std::max(1, std::min<int>(n, std::min(16u, std::thread::hardware_concurrency())));
    std::vector<std::thread> pool;
    for (int t = 1; t < nt; ++t) pool.emplace_back(work);
    work();
    for (auto& t : pool) t.join();
}

}  // namespace jpeg
}  // namespace mb

using namespace mb;
using namespace mb::jpeg;

extern "C" {

int b200_jpeg_info(const uint8_t* file, size_t nbytes, int32_t* out_height, int32_t* out_width, int32_t* out_supported) {
    return guarded([&] {
        MB_CHECK_ARG(file && out_height && out_width && out_supported, "NULL argument");
        *out_height = *out_width = 0;
        *out_supported = 0;
        Parsed p;
        try {
            parse_and_decode(file, nbytes, p);   // headers alone cannot tell (tables may be missing): decode to be sure
            *out_supported = 1;
        } catch (const Unsupported& u) {
            set_last_error(u.why);
        }
        *out_height = p.d.height;
        *out_width = p.d.width;
    });
}

int b200_jpeg_decode_batch(int device, const uint8_t* const* files, const size_t* nbytes, int n, uint8_t* const* d_out,
                           int32_t* heights, int32_t* widths, int32_t* status) {
    return guarded([&] {
        MB_CHECK_ARG(files && nbytes && d_out && heights && widths && status, "NULL argument");
        MB_CHECK_ARG(n >= 0, "n must be >= 0");
        if (n == 0) return;
        int ndev = 0;
        if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
            cudaGetLastError();
            fail(B200_ERR_NO_DEVICE, "no CUDA device available (marqo_b200 has no CPU fallback)");
        }
        MB_CHECK_ARG(device >= 0 && device < ndev, "device %d out of range", device);
        DeviceGuard g(device);
        std::vector<Parsed> imgs(n);
        std::vector<std::string> why(n);
        decode_parallel(files, nbytes, n, imgs, status, why);
        std::vector<int> ok;
        for (int i = 0; i < n; ++i) {
            heights[i] = imgs[i].d.height;
            widths[i] = imgs[i].d.width;
            if (status[i] != B200_OK) continue;
            if (heights[i] != 0 && d_out[i] == nullptr) {   // size query pass: the caller allocates and calls again
                status[i] = B200_ERR_INVALID_ARG;
                continue;
            }
            imgs[i].d.out = d_out[i];
            ok.push_back(i);
        }
        if (ok.empty()) return;
        std::vector<ImageDesc> descs;
        long long total_blocks, total_pixels, plane_bytes;
        layout_batch(imgs, ok, descs, total_blocks, total_pixels, plane_bytes);
        UniqueStream owned_stream = make_stream(cudaStreamNonBlocking);
        cudaStream_t stream = owned_stream.get();
        DeviceBuffer<ImageDesc> d_desc(descs.size());
        DeviceBuffer<int16_t> d_coef((size_t)total_blocks * 64);
        DeviceBuffer<uint8_t> d_planes((size_t)plane_bytes);
        MB_CUDA(cudaMemcpyAsync(d_desc.get(), descs.data(), descs.size() * sizeof(ImageDesc), cudaMemcpyHostToDevice,
                                stream));
        for (size_t k = 0; k < ok.size(); ++k) {
            const Parsed& p = imgs[ok[k]];
            MB_CUDA(cudaMemcpyAsync(d_coef.get() + (size_t)descs[k].block_base * 64, p.coefs.data(),
                                    p.coefs.size() * sizeof(int16_t), cudaMemcpyHostToDevice, stream));
        }
        idct_kernel<<<(unsigned)((total_blocks + 127) / 128), 128, 0, stream>>>(
            d_desc.get(), (int)descs.size(), d_coef.get(), d_planes.get(), total_blocks);
        MB_CUDA(cudaGetLastError());
        upsample_rgb_kernel<<<(unsigned)((total_pixels + 255) / 256), 256, 0, stream>>>(
            d_desc.get(), (int)descs.size(), d_planes.get(), total_pixels);
        MB_CUDA(cudaGetLastError());
        MB_CUDA(cudaStreamSynchronize(stream));
    });
}

// Test hook (NOT a product path): the same arithmetic on the host, so the CPU suite can pin it against Pillow.
int b200_debug_jpeg_decode_host(const uint8_t* file, size_t nbytes, uint8_t* out_rgb, size_t out_capacity,
                                int32_t* out_height, int32_t* out_width) {
    return guarded([&] {
        MB_CHECK_ARG(file && out_height && out_width, "NULL argument");
        Parsed p;
        try {
            parse_and_decode(file, nbytes, p);
        } catch (const Unsupported& u) {
            fail(B200_ERR_UNSUPPORTED, "%s", u.why);
        }
        ImageDesc& d = p.d;
        *out_height = d.height;
        *out_width = d.width;
        if (out_rgb == nullptr) return;
        MB_CHECK_ARG(out_capacity >= (size_t)d.height * d.width * 3, "output buffer too small");
        long long plane_bytes = 0;
        for (int c = 0; c < d.ncomp; ++c) {
            d.plane_off[c] = plane_bytes;
            plane_bytes += (long long)d.plane_w[c] * d.plane_h[c];
        }
        std::vector<uint8_t> planes((size_t)plane_bytes);
        for (int c = 0; c < d.ncomp; ++c)
            for (int by = 0; by < d.blocks_h[c]; ++by)
                for (int bx = 0; bx < d.blocks_w[c]; ++bx)
                    idct_islow(p.coefs.data() + ((size_t)d.coef_off[c] + (size_t)by * d.blocks_w[c] + bx) * 64,
                               d.q[d.qtab[c]], planes.data() + d.plane_off[c] + ((size_t)by * 8) * d.plane_w[c] + bx * 8,
                               d.plane_w[c]);
        d.out = out_rgb;
        for (int y = 0; y < d.height; ++y)
            for (int x = 0; x < d.width; ++x) output_pixel(d, planes.data(), x, y);
    });
}

}  // extern "C"
