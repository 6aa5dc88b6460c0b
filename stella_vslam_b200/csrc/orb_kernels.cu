// orb_kernels.cu -- batched feature::orb_extractor on sm_90a.
//
// Reference path (paths relative to the reference checkout):
//   orb_extractor::extract                src/stella_vslam/feature/orb_extractor.cc:28-136
//   compute_image_pyramid (cv::resize)    orb_extractor.cc:153-162
//   compute_fast_keypoints (cv::FAST)     orb_extractor.cc:164-287
//   distribute_keypoints                  orb_extractor.cc:289-329
//   ic_angle / compute_orb_descriptor     feature/orb_impl.cc:68-91, 93-154
//   cv::GaussianBlur 7x7 sigma 2          orb_extractor.cc:103
//
// Design (see DESIGN.md): every kernel takes a batch of same-sized frames (blockIdx.y = frame).  The order-dependent
// parts of the reference are restated as order-free reductions: FAST candidates are never materialised as a list --
// each surviving corner does one 64-bit atomicMax (score, inverse scan order) into its selection-grid cell, which is
// exactly "first candidate with strictly greatest response" (orb_extractor.cc:314-323).  Keypoints are then emitted
// by an ordered compaction of the grid (level-major, cell-index order = the reference's output order).
//
// Integer work is bit-exact by construction; the only floating point (fastAtan2, util::cos/sin, the rBRIEF rotation,
// pt *= scale) uses explicit round-to-nearest intrinsics, never FMA (this file is also compiled with -fmad=false).
#include <cuda.h>

#include <algorithm>
#include <cmath>
#include <new>
#include <vector>

#include "camera_model.cuh"
#include "common.cuh"
#include "staging.cuh"
#include "track_chain.cuh"
#include "util_trig.cuh"

namespace b200 {
namespace orb {

constexpr int kMaxLevels = 16;
constexpr int kBorder = 19;       // orb_extractor.h:107 orb_patch_radius_
constexpr int kCell = 64;         // orb_extractor.cc:173
constexpr int kOverlap = 6;       // orb_extractor.cc:172
constexpr int kTileMax = kCell + kOverlap;  // 70
constexpr int kTilePitch = 80;    // smem row pitch of a FAST tile (multiple of 16 for TMA boxes)

struct LevelGeom {
    int w, h, pitch;
    unsigned long long offset;    // byte offset of the level inside one frame's pyramid (level 0: unused)
    float sf;                     // scale_factors_[l]
    int nx, ny;                   // selection grid (orb_extractor.cc:293-294)
    double delta_x, delta_y;      // orb_extractor.cc:295-296
    int grid_base;                // first grid cell of this level in the per-frame grid array
    int ncols;                    // FAST cell columns (for the scan-order key)
    float size;                   // (float)(unsigned)(31 * sf)  orb_extractor.cc:274
    int tab_x, tab_y;             // offsets into the resize tables (level l is resampled from level l-1)
};

struct Geom {
    int num_levels;
    int grid_cells;               // selection-grid cells per frame (all levels)
    int ini_thr, min_thr;
    LevelGeom lv[kMaxLevels];
};

struct CellDesc {                 // one FAST cell (orb_extractor.cc:199-217)
    unsigned short level, i, j, min_x, min_y, w, h, pad;
};

struct RawKp {                    // keypoint before orientation/description
    short x, y;                   // level coordinates (border already added)
    unsigned char m;              // FAST m value; response = m - 1
    unsigned char level;
    unsigned short pad;
};

struct ResizeTap {                // per destination column/row: source index and the two Q11 weights
    short ofs, w0, w1, pad;
};

// ---------------------------------------------------------------------------------------------------------------
// image access helpers: level 0 aliases the caller's frames (orb_extractor.cc:154), levels >= 1 live in the pyramid
// ---------------------------------------------------------------------------------------------------------------
struct Images {
    const unsigned char* img0;
    unsigned long long pitch0, fstride0;
    unsigned char* pyr;
    unsigned long long pyr_fstride;
};

__device__ __forceinline__ const unsigned char* level_ptr(const Images& im, const Geom& g, int level, int frame, int* pitch) {
    if (level == 0) {
        *pitch = (int)im.pitch0;
        return im.img0 + (size_t)frame * im.fstride0;
    }
    *pitch = g.lv[level].pitch;
    return im.pyr + (size_t)frame * im.pyr_fstride + g.lv[level].offset;
}

// ---------------------------------------------------------------------------------------------------------------
// TMA: one 3-D tensor map (x, y, frame) per pyramid level; a FAST cell tile is ONE bulk-tensor copy, out-of-image bytes are
// zero-filled by the hardware.  (cp.async.bulk.tensor -> UTMALDG; completion through an mbarrier transaction count.)
// ---------------------------------------------------------------------------------------------------------------
struct TmapSet {
    CUtensorMap m[kMaxLevels];
};

__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");  // make the init visible to the async proxy
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* tmap, int x, int y, int z, unsigned long long* bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(reinterpret_cast<unsigned long long>(tmap)), "r"(x), "r"(y), "r"(z), "r"(smem_u32(bar))
                 : "memory");
}

// ---------------------------------------------------------------------------------------------------------------
// K1: cv::resize(INTER_LINEAR) level l-1 -> l, fixed point (OpenCV resize.cpp HResizeLinear/VResizeLinear, 11 bits)
// ---------------------------------------------------------------------------------------------------------------
// One thread produces a strip of 4 columns x kRzRows rows: the x taps are loaded once, and the horizontally interpolated value
// of every source row is computed once and reused by the (usually two) output rows that blend it -- half the gathers and
// multiplies of a row-at-a-time kernel.  Source bytes come straight from L1/L2 (a shared-memory staged variant, measured on an
// earlier GPU target and not on the H100, was slower: the tile fill + barrier cost more than the cached gathers).
constexpr int kRzRows = 8;

__global__ void __launch_bounds__(128) resize_kernel(const __grid_constant__ Geom g, Images im, const ResizeTap* __restrict__ taps, int level) {
    const LevelGeom& L = g.lv[level];
    const int frame = blockIdx.z;
    int spitch;
    const unsigned char* src = level_ptr(im, g, level - 1, frame, &spitch);
    unsigned char* dst = im.pyr + (size_t)frame * im.pyr_fstride + L.offset;
    const int sw = g.lv[level - 1].w, sh = g.lv[level - 1].h;
    const int dxq = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    const int dy0 = blockIdx.y * kRzRows;
    if (dxq >= L.pitch) return;
    const int n_valid = min(4, L.w - dxq);  // <= 0 in the padding columns (written as zero)
    // The padding columns re-use the taps of the last valid column (in-bounds loads, no per-column predicates); their bytes are
    // masked to zero at the store.
    const unsigned store_mask = n_valid >= 4 ? 0xFFFFFFFFu : (n_valid <= 0 ? 0u : ((1u << (8 * n_valid)) - 1u));
    int ofs[4], ofs1[4];
    unsigned w01[4];  // w0 | w1 << 16: the horizontal tap pair as the 16-bit operand of one DP2A
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const ResizeTap t = taps[L.tab_x + min(dxq + k, L.w - 1)];
        ofs[k] = t.ofs;
        ofs1[k] = min((int)t.ofs + 1, sw - 1);  // weight 0 there
        w01[k] = ((unsigned)t.w0 & 0xFFFFu) | ((unsigned)t.w1 << 16);
    }
    int rowA = -1, rowB = -1;  // clipped source rows whose horizontal interpolation is cached
    unsigned hA[4] = {0, 0, 0, 0}, hB[4] = {0, 0, 0, 0};
    auto hrow = [&](int sy, unsigned (&h)[4]) {
        const unsigned char* r = src + (size_t)sy * spitch;
#pragma unroll
        for (int k = 0; k < 4; ++k) h[k] = __dp2a_lo(w01[k], (unsigned)r[ofs[k]] | ((unsigned)r[ofs1[k]] << 8), 0u) >> 4;
    };
    const int dy_end = min(dy0 + kRzRows, L.h);
    unsigned char* drow = dst + (size_t)dy0 * L.pitch + dxq;
    for (int dy = dy0; dy < dy_end; ++dy, drow += L.pitch) {
        const ResizeTap ty = taps[L.tab_y + dy];
        const int s0 = min(max((int)ty.ofs, 0), sh - 1), s1 = min(max((int)ty.ofs + 1, 0), sh - 1);  // rows clipped like OpenCV
        if (s0 != rowA) {
            if (s0 == rowB) {
#pragma unroll
                for (int k = 0; k < 4; ++k) hA[k] = hB[k];
            } else {
                hrow(s0, hA);
            }
            rowA = s0;
        }
        if (s1 != rowB) {
            if (s1 == rowA) {
#pragma unroll
                for (int k = 0; k < 4; ++k) hB[k] = hA[k];
            } else {
                hrow(s1, hB);
            }
            rowB = s1;
        }
        // ((b0 * S0) >> 16) as the high half of (b0 << 16) * S0: weights are in [0, 2048] and S in [0, 32640], so everything is
        // non-negative and the result (<= 255: the weights of a pair sum to 2048) needs no saturation
        const unsigned b0 = (unsigned)(int)ty.w0 << 16, b1 = (unsigned)(int)ty.w1 << 16;
        unsigned out = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) out |= ((__umulhi(b0, hA[k]) + __umulhi(b1, hB[k]) + 2u) >> 2) << (8 * k);
        *reinterpret_cast<unsigned*>(drow) = out & store_mask;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// K2: FAST-9/16 + 3x3 NMS per 64-px cell with the per-cell threshold retry, mask tests, and the selection-grid
//     arg-max.  One block per (cell, frame).
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool has_run9(unsigned m16) {
    unsigned m = m16 | (m16 << 16);
    unsigned x = m & (m >> 1);
    x &= x >> 2;
    x &= x >> 4;
    x &= m >> 8;
    return (x & 0xFFFFu) != 0;
}

// circle offsets in a tile of pitch kTilePitch, OpenCV order (fast.cpp makeOffsets, patternSize 16)
#define FAST_OFF(k, P)                                                                                              \
    ((k) == 0 ? 3 * (P) : (k) == 1 ? 3 * (P) + 1 : (k) == 2 ? 2 * (P) + 2 : (k) == 3 ? (P) + 3 : (k) == 4 ? 3      \
     : (k) == 5 ? -(P) + 3 : (k) == 6 ? -2 * (P) + 2 : (k) == 7 ? -3 * (P) + 1 : (k) == 8 ? -3 * (P)              \
     : (k) == 9 ? -3 * (P)-1 : (k) == 10 ? -2 * (P)-2 : (k) == 11 ? -(P)-3 : (k) == 12 ? -3                        \
     : (k) == 13 ? (P)-3 : (k) == 14 ? 2 * (P)-2 : 3 * (P)-1)

__device__ __forceinline__ bool mask_zero(const unsigned char* mask, unsigned long long mask_pitch, unsigned y, unsigned x, float sf) {
    // orb_extractor.cc:168-170: mask.at<uchar>(y * scale_factor, x * scale_factor): float product, truncation
    const int r = (int)__fmul_rn((float)y, sf), c = (int)__fmul_rn((float)x, sf);
    return mask[(size_t)r * mask_pitch + c] == 0;
}

// Exact FAST score map for FOUR horizontally adjacent pixels (two u16x2 lane pairs: even = px 0,2 / odd = px 1,3).
// m = max( v - min_s max_{arc s} p ,  max_s min_{arc s} p - v )  over the 16 arcs of 9 contiguous circle pixels, computed with
// the packed 3-input min/max (VIMNMX3.U16x2): 16 window-3 + 16 window-9 + 8 reduction ops per polarity and lane
// pair.  Working on the raw pixel values (not on differences) keeps everything unsigned and never negates a min/max
// result (see the ptxas note in DESIGN.md).  Returns max(m - t_low, 0) per pixel, packed as 4 bytes.
// (An exact early-out on the four even antipodal pairs -- every 9-arc holds one pixel of each pair -- was measured on an
// earlier GPU target: it never retires a whole warp on the bench stream and cost time, so the arcs are always evaluated.)
__device__ __forceinline__ unsigned fast_m4(const unsigned (&w)[7][3], unsigned neg_tlow2) {
    // circle offsets (dx, dy) in OpenCV order; row index = dy + 3, window = 4 bytes starting at column c0 + dx
    constexpr int DX[16] = {0, 1, 2, 3, 3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1};
    constexpr int DY[16] = {3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1, 0, 1, 2, 3};
    unsigned pe[16], po[16];
    const unsigned ve = __byte_perm(w[3][1], 0, 0x4240), vo = __byte_perm(w[3][1], 0, 0x4341);
    auto extract = [&](int k) {
        const int dx = DX[k], r = DY[k] + 3;
        unsigned x;
        if (dx == 0) x = w[r][1];
        else if (dx > 0) x = __byte_perm(w[r][1], w[r][2], 0x3210 + 0x1111 * dx);
        else x = __byte_perm(w[r][0], w[r][1], 0x3210 + 0x1111 * (4 + dx));
        pe[k] = __byte_perm(x, 0, 0x4240);  // pixels 0 and 2 as u16x2
        po[k] = __byte_perm(x, 0, 0x4341);  // pixels 1 and 3
    };
#pragma unroll
    for (int k = 0; k < 16; ++k) extract(k);
    unsigned res[2];
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        const unsigned* p = half ? po : pe;
        const unsigned v = half ? vo : ve;
        unsigned mx3[16], mn3[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            mx3[k] = __vimax3_u16x2(p[k], p[(k + 1) & 15], p[(k + 2) & 15]);
            mn3[k] = __vimin3_u16x2(p[k], p[(k + 1) & 15], p[(k + 2) & 15]);
        }
        unsigned mx9[16], mn9[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            mx9[k] = __vimax3_u16x2(mx3[k], mx3[(k + 3) & 15], mx3[(k + 6) & 15]);
            mn9[k] = __vimin3_u16x2(mn3[k], mn3[(k + 3) & 15], mn3[(k + 6) & 15]);
        }
        // a = min over arcs of (max over the arc), b = max over arcs of (min over the arc)
        unsigned a = __vimin3_u16x2(mx9[0], mx9[1], mx9[2]), b = __vimax3_u16x2(mn9[0], mn9[1], mn9[2]);
#pragma unroll
        for (int k = 3; k < 15; k += 2) {
            a = __vimin3_u16x2(a, mx9[k], mx9[k + 1]);
            b = __vimax3_u16x2(b, mn9[k], mn9[k + 1]);
        }
        a = __vminu2(a, mx9[15]);
        b = __vmaxu2(b, mn9[15]);
        const unsigned dark = __vsub2(v, a), bright = __vsub2(b, v);       // signed 16-bit lanes, |.| <= 255
        const unsigned m = __vimax_s16x2_relu(dark, bright);               // max(dark, bright, 0)
        res[half] = __viaddmax_s16x2_relu(m, neg_tlow2, 0u);               // max(m - t_low, 0)
    }
    return __byte_perm(res[0], res[1], 0x6240);  // bytes: px0, px1, px2, px3
}

// Candidate test for 4 pixels (exact superset of m > t_low).  Every 9-arc of the circle contains one pixel of each antipodal pair
// {k, k+8}, hence   max_arcs min_arc p <= min_pairs max(p_k, p_k+8)   and   min_arcs max_arc p >= max_pairs min(p_k, p_k+8).
// With the two compass pairs this bounds m from above; a pixel whose bound does not exceed t_low stores 0 without the arc
// evaluation.  ~10 % of the pixels of a natural frame pass at t_low = 7, so the arcs are evaluated for those only (fast_score1).
// Returns a 4-bit mask.
__device__ __forceinline__ unsigned fast_candidates4(const unsigned (&w)[7][3], unsigned tlow2) {
    const unsigned x0 = w[6][1], x8 = w[0][1];                                                          // (0, +3), (0, -3)
    const unsigned x4 = __byte_perm(w[3][1], w[3][2], 0x6543), x12 = __byte_perm(w[3][0], w[3][1], 0x4321);  // (+3, 0), (-3, 0)
    unsigned r[2];
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        const unsigned sel = half ? 0x4341u : 0x4240u;  // pixels (1, 3) / (0, 2) as u16x2
        const unsigned p0 = __byte_perm(x0, 0, sel), p8 = __byte_perm(x8, 0, sel), p4 = __byte_perm(x4, 0, sel), p12 = __byte_perm(x12, 0, sel);
        const unsigned v = __byte_perm(w[3][1], 0, sel);
        const unsigned hi = __vminu2(__vmaxu2(p0, p8), __vmaxu2(p4, p12));
        const unsigned lo = __vmaxu2(__vminu2(p0, p8), __vminu2(p4, p12));
        // bound > t_low  <=>  hi > v + t_low  or  v > lo + t_low.  Only unsigned lane max and XOR: the signed packed subtract / relu
        // forms of this test (vsub2 + vimax_s16x2_relu + viaddmax_s16x2_relu) came out wrong in this context when built for sm_100a (tools/fast_probe)
        const unsigned vt = v + tlow2, lot = lo + tlow2;  // lanes <= 510: no carry between them
        r[half] = (__vmaxu2(hi, vt) ^ vt) | (__vmaxu2(v, lot) ^ lot);
    }
    return ((r[0] & 0xFFFFu) ? 1u : 0u) | ((r[1] & 0xFFFFu) ? 2u : 0u) | ((r[0] >> 16) ? 4u : 0u) | ((r[1] >> 16) ? 8u : 0u);
}

// Exact FAST-9/16 score of ONE pixel at tile position p (same definition as fast_m4, scalar 3-input min/max): max(m - t_low, 0).
__device__ __forceinline__ int fast_score1(const unsigned char* __restrict__ p, int t_low) {
    constexpr int OFF[16] = {3 * kTilePitch,     3 * kTilePitch + 1,  2 * kTilePitch + 2,  kTilePitch + 3,  3,  -kTilePitch + 3, -2 * kTilePitch + 2, -3 * kTilePitch + 1,
                             -3 * kTilePitch,    -3 * kTilePitch - 1, -2 * kTilePitch - 2, -kTilePitch - 3, -3, kTilePitch - 3,  2 * kTilePitch - 2,  3 * kTilePitch - 1};
    // Both polarities in one pass of packed 16-bit lanes: low half = the ring pixel c, high half = 255 - c.  "min over the 16 arcs of
    // the arc maximum" of the low halves is a (dark corners); of the high halves it is 255 - b, b = max over arcs of the arc minimum
    // (bright corners).  40 VIMNMX3.S16x2 instead of 96 scalar min/max.
    unsigned c[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) c[k] = (unsigned)p[OFF[k]] * 0xFFFF0001u + 0x00FF0000u;  // c | (255 - c) << 16
    const int v = p[0];
    unsigned mx3[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) mx3[k] = __vimax3_s16x2(c[k], c[(k + 1) & 15], c[(k + 2) & 15]);
    unsigned ab = 0x00FF00FFu;
#pragma unroll
    for (int k = 0; k < 16; k += 2)  // two arcs per 3-input minimum
        ab = __vimin3_s16x2(ab, __vimax3_s16x2(mx3[k], mx3[(k + 3) & 15], mx3[(k + 6) & 15]),
                            __vimax3_s16x2(mx3[k + 1], mx3[(k + 4) & 15], mx3[(k + 7) & 15]));
    const int a = (int)(ab & 0xFFFFu), b = 255 - (int)(ab >> 16);
    // max(m - t_low, 0) with m = max(v - a, b - v, 0).  The dark and the bright excess cannot both be positive (two 9-arcs of a
    // 16-circle share pixels), so the result is their sum: no max of a difference is formed, which keeps ptxas from emitting
    // VIADDMNMX with a negated addend (measured wrong when built for sm_100a, like the VIMNMX3 case in DESIGN.md).
    const int at = a + t_low, vt = v + t_low;
    return (max(v, at) - at) + (max(b, vt) - vt);
}

constexpr int kFastThreads = 256;
constexpr int kTileRows = kTileMax + 2;  // 72
constexpr int kRawPitch = 96;            // TMA box width: the box must start on a 16-byte boundary of the row (x0 = 16 + 64 j),
                                         // i.e. 2 bytes left of the tile origin (x = 18 + 64 j), and cover 82 bytes

// kUseTma: the tile arrives through the level's tensor map (needs a 16-byte aligned base and 16-byte multiples as
// strides, always true for the pyramid arena; checked on the host for the caller's level-0 frames).  Otherwise the same
// tile is assembled with ordinary loads.
template <bool kUseTma>
__global__ void __launch_bounds__(kFastThreads) fast_cells_kernel(const __grid_constant__ Geom g, const __grid_constant__ TmapSet tmaps, Images im,
                                                                  const CellDesc* __restrict__ cells, const unsigned char* __restrict__ mask,
                                                                  unsigned long long mask_pitch, unsigned long long* __restrict__ grid,
                                                                  int arena_frame0, int* __restrict__ raw_corners) {
    // tile column c holds cell column c - 1 (so the first candidate column, lx = 3, is 4-byte aligned); pitch 80
    __shared__ __align__(16) unsigned char tile[kTileRows * kTilePitch];
    __shared__ __align__(16) unsigned char mmap[kTileRows * kTilePitch];
    __shared__ __align__(128) unsigned char raw[kUseTma ? kTileRows * kRawPitch : 16];  // TMA landing zone
    __shared__ __align__(8) unsigned long long tma_bar;
    __shared__ int skip;
    __shared__ unsigned short cand[(kTileMax - 6) * (kTileMax - 6)];  // (row << 8 | tile column) of the pixels that need the arc evaluation
    __shared__ int n_cand;

    const CellDesc cd = cells[blockIdx.x];
    const int frame = blockIdx.y;
    const int level = cd.level;
    const LevelGeom& L = g.lv[level];
    const int cw = cd.w, ch = cd.h;
    const int tid = threadIdx.x;

    if (tid == 0) {
        int s = 0;
        if (mask) {  // orb_extractor.cc:219-225: skip the cell if one of its corners is masked
            const unsigned max_x = cd.min_x + cw, max_y = cd.min_y + ch;
            s = mask_zero(mask, mask_pitch, cd.min_y, cd.min_x, L.sf) || mask_zero(mask, mask_pitch, max_y, cd.min_x, L.sf)
                || mask_zero(mask, mask_pitch, cd.min_y, max_x, L.sf) || mask_zero(mask, mask_pitch, max_y, max_x, L.sf);
        }
        skip = s;
        n_cand = 0;
    }
    if constexpr (kUseTma) {
        // one elected thread: arm the mbarrier with the tile's byte count and issue the bulk-tensor copy of the 80 x 72 box
        // whose origin is (min_x - 1, min_y, frame); bytes outside the image come back as zeros
        if (tid == 0) {
            mbar_init(&tma_bar, 1);
            mbar_expect_tx(&tma_bar, kTileRows * kRawPitch);
            // min_x - 3 = 16 + 64 j.  Levels >= 1 are described over the whole arena, level 0 over this call's frames.
            tma_load_3d(raw, &tmaps.m[level], (int)cd.min_x - 3, (int)cd.min_y, frame + (level ? arena_frame0 : 0), &tma_bar);
        }
        __syncthreads();  // barrier initialised (and skip written) before anybody polls it
        mbar_wait(&tma_bar, 0);
        // re-pitch into the compute tile, shifting by the 2 alignment bytes: tile byte c = raw byte c + 2
        for (int idx = tid; idx < kTileRows * (kTilePitch / 4); idx += kFastThreads) {
            const int y = idx / (kTilePitch / 4), q = idx - y * (kTilePitch / 4);
            const unsigned* rw = reinterpret_cast<const unsigned*>(raw + y * kRawPitch) + q;
            reinterpret_cast<unsigned*>(tile)[idx] = __funnelshift_r(rw[0], rw[1], 16);
            reinterpret_cast<unsigned*>(mmap)[idx] = 0u;
        }
        __syncthreads();
    } else {
        int pitch;
        const unsigned char* src = level_ptr(im, g, level, frame, &pitch);
        src += (size_t)cd.min_y * pitch + cd.min_x;
        // rows 0..ch-1 of the cell -> tile rows 0..ch-1; two extra zero rows keep the 4-row groups in bounds
        for (int idx = tid; idx < kTileRows * (kTilePitch / 4); idx += kFastThreads) {
            const int y = idx / (kTilePitch / 4), c4 = (idx - y * (kTilePitch / 4)) * 4;
            unsigned v = 0;
            if (y < ch) {
#pragma unroll
                for (int b = 0; b < 4; ++b) {
                    const int x = c4 + b - 1;  // cell column
                    if (x >= 0 && x < cw) v |= (unsigned)src[(size_t)y * pitch + x] << (8 * b);
                }
            }
            reinterpret_cast<unsigned*>(tile)[idx] = v;
            reinterpret_cast<unsigned*>(mmap)[idx] = 0u;
        }
        __syncthreads();
    }
    if (skip) return;

    const int t_low = min(g.ini_thr, g.min_thr);
    const unsigned neg_tlow2 = (unsigned)((-t_low) & 0xFFFF) * 0x10001u;
    // phase 1a: candidate test.  thread = (word column wq, group of 4 rows); candidate columns lx in [3, cw-4] <=> tile column lx+1.
    // A pixel can only be a corner at threshold t if one pixel of each compass pair {(0,+3),(0,-3)} and {(+3,0),(-3,0)} differs from
    // it by more than t (every 9-arc holds one pixel of each antipodal pair), whatever the sign: a superset of the u16x2 bound
    // test above (10.7 % instead of 9.7 % of the bench stream's pixels pass at t = 7) that runs at BYTE width -- sm_90a has no
    // native byte min/max or compare (the video intrinsics expand to PRMT / LOP3 sequences in the SASS) but it does have
    // VABSDIFF4, and "|d| > t" on four bytes is three logic/add operations.  20 instead of 46 instructions per four pixels.
    if (t_low <= 126) {
        const int wq = tid & 15, rg = tid >> 4;       // 16 word columns x 16 row groups
        const int c0 = 4 + 4 * wq;                    // tile column of the first pixel of the word
        const int lx0 = c0 - 1;                       // its cell column
        const int y0 = 3 + 4 * rg;                    // first candidate row of the group
        if (lx0 <= cw - 4 && y0 <= ch - 4) {
            const unsigned c7f = (unsigned)(0x7F - t_low) * 0x01010101u;
            auto gt = [&](unsigned d) { return (((d & 0x7F7F7F7Fu) + c7f) | d) & 0x80808080u; };  // bit 7 of byte b: d_b > t_low
            unsigned ctr[10];  // centre words of rows y0-3 .. y0+6
#pragma unroll
            for (int r = 0; r < 10; ++r) ctr[r] = *reinterpret_cast<const unsigned*>(tile + (y0 - 3 + r) * kTilePitch + c0);
            unsigned acc = 0;  // byte b (pixel), bit i (row): candidate
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const unsigned* row = reinterpret_cast<const unsigned*>(tile + (y0 + i) * kTilePitch + c0 - 4);
                const unsigned v = ctr[i + 3];
                const unsigned p4 = __byte_perm(v, row[2], 0x6543), p12 = __byte_perm(row[0], v, 0x4321);  // (+3, 0), (-3, 0)
                const unsigned gbits = (gt(__vabsdiffu4(ctr[i + 6], v)) | gt(__vabsdiffu4(ctr[i], v))) & (gt(__vabsdiffu4(p4, v)) | gt(__vabsdiffu4(p12, v)));
                acc |= gbits >> (7 - i);
            }
            // pixels of this word that are candidates: lx0 + b <= cw - 4; rows y0 + i <= ch - 4
            const int nvalid = min(4, cw - 3 - lx0), nrows = min(4, ch - 3 - y0);
            acc &= (0xFFFFFFFFu >> (32 - 8 * nvalid)) & (((1u << nrows) - 1u) * 0x01010101u);
            if (acc) {
                // sixteen predicated stores at prefix-popcount offsets instead of a loop over the set bits: the loop ran as long as the
                // fullest thread of the warp
                int pos = atomicAdd(&n_cand, __popc(acc));
                const unsigned enc0 = (unsigned)((y0 << 8) | c0);
#pragma unroll
                for (int b = 0; b < 4; ++b) {
                    const unsigned nib = (acc >> (8 * b)) & 0xFu;  // rows y0 .. y0 + 3 of pixel c0 + b
#pragma unroll
                    for (int i = 0; i < 4; ++i)
                        if ((nib >> i) & 1u) cand[pos + __popc(nib & ((1u << i) - 1u))] = (unsigned short)(enc0 + (unsigned)((i << 8) | b));
                    pos += __popc(nib);
                }
            }
        }
    } else {
        const int wq = tid & 15, rg = tid >> 4;
        const int c0 = 4 + 4 * wq;
        const int lx0 = c0 - 1;
        const int y0 = 3 + 4 * rg;
        if (lx0 <= cw - 4 && y0 <= ch - 4) {
            unsigned w[10][3];
#pragma unroll
            for (int r = 0; r < 10; ++r) {
                const int y = y0 - 3 + r;  // <= ch + 2 < kTileMax + 2
                const unsigned* row = reinterpret_cast<const unsigned*>(tile + y * kTilePitch + c0 - 4);
                w[r][0] = row[0];
                w[r][1] = row[1];
                w[r][2] = row[2];
            }
            const int nvalid = min(4, cw - 3 - lx0);
            const unsigned keep = (1u << nvalid) - 1u;
            unsigned bits = 0;  // 4 rows x 4 pixels
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                if (y0 + i <= ch - 4) {
                    unsigned ww[7][3];
#pragma unroll
                    for (int r = 0; r < 7; ++r) {
                        ww[r][0] = w[i + r][0];
                        ww[r][1] = w[i + r][1];
                        ww[r][2] = w[i + r][2];
                    }
                    bits |= (fast_candidates4(ww, (unsigned)t_low * 0x10001u) & keep) << (4 * i);
                }
            }
            if (bits) {
                int pos = atomicAdd(&n_cand, __popc(bits));
                while (bits) {
                    const int k = __ffs(bits) - 1;
                    bits &= bits - 1;
                    cand[pos++] = (unsigned short)(((y0 + (k >> 2)) << 8) | (c0 + (k & 3)));
                }
            }
        }
    }
    __syncthreads();
    // phase 1b: exact score of the candidates (the score map is zero everywhere else)
    {
        const int n = n_cand;
        for (int i = tid; i < n; i += kFastThreads) {
            const int e = cand[i], y = e >> 8, c = e & 0xFF;
            mmap[y * kTilePitch + c] = (unsigned char)fast_score1(tile + y * kTilePitch + c, t_low);
        }
    }
    __syncthreads();
    // phase 2: strict 3x3 local maximum of m (threshold independent), per-cell threshold choice
    //          (orb_extractor.cc:228-235: retry the whole cell at min_fast_thr only if it is empty at ini_fast_thr).
    // Only the candidates of phase 1a can have a non-zero score, so the test walks the compacted candidate list (~10 % of the
    // pixels) instead of the score map: one thread per candidate, eight neighbour bytes each.
    const int ini_rel = g.ini_thr - t_low, min_rel = g.min_thr - t_low;  // thresholds relative to the stored m - t_low
    const int n_c = n_cand;
    unsigned kept = 0;  // bit `it`: this thread's it-th candidate is a strict local maximum with a usable score
    bool any_ini = false;
    {
        int it = 0;
        for (int i = tid; i < n_c; i += kFastThreads, ++it) {
            const int e = cand[i];
            const unsigned char* p = mmap + (e >> 8) * kTilePitch + (e & 0xFF);
            const int mv = p[0];
            // stored value is m - t_low; a keypoint needs score m - 1 >= 1
            if (mv == 0 || mv + t_low < 2) continue;
            const bool is_max = mv > p[-1] && mv > p[1] && mv > p[-kTilePitch - 1] && mv > p[-kTilePitch] && mv > p[-kTilePitch + 1]
                                && mv > p[kTilePitch - 1] && mv > p[kTilePitch] && mv > p[kTilePitch + 1];
            if (is_max) {
                kept |= 1u << it;  // (at most 64 * 64 / 256 = 16 candidates per thread)
                any_ini |= (mv > ini_rel);
            }
        }
    }
    const int cell_has_ini = __syncthreads_or(any_ini);
    const int thr_rel = cell_has_ini ? ini_rel : min_rel;
    // phase 3: mask test per keypoint, selection-grid cell, ordered arg-max via 64-bit atomicMax
    int n_raw = 0;  // FAST corners this thread hands to distribute_keypoints (the C of SURVEY 8d's byte formulas)
    while (kept) {
        const int it = __ffs(kept) - 1;
        kept &= kept - 1;
        const int e = cand[tid + it * kFastThreads], y = e >> 8, c = e & 0xFF;
        const int mrel = mmap[y * kTilePitch + c];
        if (mrel <= thr_rel) continue;
        const int mv = mrel + t_low;
        const int lx = c - 1, ly = y;
        // keypt.pt += (j*64, i*64) (orb_extractor.cc:241-244): coordinates relative to the (19,19) border origin
        const int px = lx + cd.j * kCell, py = ly + cd.i * kCell;
        if (mask && mask_zero(mask, mask_pitch, (unsigned)(kBorder + py), (unsigned)(kBorder + px), L.sf)) continue;
        const unsigned ix = (unsigned)((double)(float)px / L.delta_x);  // orb_extractor.cc:303-305
        const unsigned iy = (unsigned)((double)(float)py / L.delta_y);
        const unsigned cell = ix + iy * (unsigned)L.nx;
        const unsigned order = ((unsigned)(cd.i * L.ncols + cd.j) << 14) | ((unsigned)ly << 7) | (unsigned)lx;
        const unsigned long long val = ((unsigned long long)mv << 32) | (unsigned long long)(0xFFFFFFFFu - order);
        atomicMax(grid + (size_t)frame * g.grid_cells + L.grid_base + cell, val);
        ++n_raw;
    }
    if (raw_corners) {
#pragma unroll
        for (int s2 = 16; s2 > 0; s2 >>= 1) n_raw += __shfl_xor_sync(0xFFFFFFFFu, n_raw, s2);
        if ((tid & 31) == 0 && n_raw) atomicAdd(raw_corners + frame, n_raw);
    }
}

// ---------------------------------------------------------------------------------------------------------------
// K3: ordered compaction of the selection grid -> per-frame raw keypoint list in the reference's output order
//     (level-major, grid-cell index ascending; orb_extractor.cc:309-326, 132-135).  One block per (level, frame).
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) select_kernel(const __grid_constant__ Geom g, const unsigned long long* __restrict__ grid,
                                                     RawKp* __restrict__ raw, int raw_stride, int* __restrict__ counts,
                                                     int* __restrict__ level_counts) {
    __shared__ int warp_sums[8];
    __shared__ int running;
    const int level = blockIdx.x, frame = blockIdx.y;
    const LevelGeom& L = g.lv[level];
    const unsigned long long* gf = grid + (size_t)frame * g.grid_cells;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    // offset = keypoints of all lower levels
    int below = 0;
    for (int base = 0; base < L.grid_base; base += blockDim.x) {
        const int i = base + tid;
        below += __syncthreads_count(i < L.grid_base && gf[i] != 0ull);
    }
    if (tid == 0) running = below;
    __syncthreads();
    const int n_cells = L.nx * L.ny;
    for (int base = 0; base < n_cells; base += blockDim.x) {
        const int i = base + tid;
        const unsigned long long v = (i < n_cells) ? gf[L.grid_base + i] : 0ull;
        const bool has = v != 0ull;
        const unsigned bal = __ballot_sync(0xFFFFFFFFu, has);
        if (lane == 0) warp_sums[wid] = __popc(bal);
        __syncthreads();
        int off = running;
        for (int w = 0; w < wid; ++w) off += warp_sums[w];
        if (has) {
            const int pos = off + __popc(bal & ((1u << lane) - 1u));
            const unsigned order = 0xFFFFFFFFu - (unsigned)(v & 0xFFFFFFFFull);
            const int lx = order & 127, ly = (order >> 7) & 127, cidx = order >> 14;
            const int ci = cidx / L.ncols, cj = cidx - ci * L.ncols;
            RawKp k;
            k.x = (short)(kBorder + cj * kCell + lx);
            k.y = (short)(kBorder + ci * kCell + ly);
            k.m = (unsigned char)(v >> 32);
            k.level = (unsigned char)level;
            k.pad = 0;
            raw[(size_t)frame * raw_stride + pos] = k;
        }
        __syncthreads();
        if (tid == 0) {
            int s = 0;
            for (int w = 0; w < 8; ++w) s += warp_sums[w];
            running += s;
        }
        __syncthreads();
    }
    if (tid == 0) {
        level_counts[frame * kMaxLevels + level] = running - below;
        if (level == g.num_levels - 1) counts[frame] = running;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// K4: cv::GaussianBlur 7x7 sigma 2 REFLECT_101 on u8, OpenCV's fixed-point path: Q8.8 taps {18,34,48,56,48,34,18},
//     16-bit horizontal pass, Q16.16 vertical pass, round to nearest.  One block per 64x32 output tile.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kBlurTW = 64, kBlurTH = 32;
constexpr int kBlurInW = kBlurTW + 8;     // input tile bytes per row: columns x0-4 .. x0+67 (18 aligned words)
constexpr int kBlurInH = kBlurTH + 6;     // rows y0-3 .. y0+34

__device__ __forceinline__ int reflect101(int i, int n) {
    if (i < 0) i = -i;
    if (i >= n) i = 2 * n - 2 - i;
    return min(max(i, 0), n - 1);  // (levels narrower than 4 px never carry keypoints)
}

// Horizontal 7-tap pass for 4 consecutive outputs with two dp4a each: taps {18,34,48,56} on bytes c-3..c and
// {48,34,18,0} on bytes c+1..c+4.  w0..w2 are the aligned words holding tile bytes 4q .. 4q+11 (output c = 4q+k <-> byte 4q+k+4).
__device__ __forceinline__ void blur_h4(unsigned w0, unsigned w1, unsigned w2, unsigned (&h)[4]) {
    constexpr unsigned TA = 18u | (34u << 8) | (48u << 16) | (56u << 24);
    constexpr unsigned TB = 48u | (34u << 8) | (18u << 16);
    h[0] = __dp4a(__byte_perm(w0, w1, 0x4321), TA, __dp4a(__byte_perm(w1, w2, 0x4321), TB, 0u));
    h[1] = __dp4a(__byte_perm(w0, w1, 0x5432), TA, __dp4a(__byte_perm(w1, w2, 0x5432), TB, 0u));
    h[2] = __dp4a(__byte_perm(w0, w1, 0x6543), TA, __dp4a(__byte_perm(w1, w2, 0x6543), TB, 0u));
    h[3] = __dp4a(w1, TA, __dp4a(w2, TB, 0u));
}

// ---------------------------------------------------------------------------------------------------------------
// K5: IC-angle orientation on the un-blurred level + rBRIEF on the blurred level + scale correction.
//     One warp per keypoint; lane u-15 sums column u of the disc, lane i produces descriptor byte i.
// ---------------------------------------------------------------------------------------------------------------
__constant__ __align__(16) signed char c_pattern[1024] = {
#include "orb_pattern.inc"
};
__constant__ int c_umax[16] = {15, 15, 15, 15, 14, 14, 14, 13, 13, 12, 11, 10, 9, 8, 6, 3};  // orb_impl.cc:51-66

// cv::fastAtan2 scalar path (OpenCV mathfuncs_core atan_f32), degrees
__device__ __forceinline__ float fast_atan2_deg(float y, float x) {
    const float rad2deg = (float)(180 / 3.1415926535897932384626433832795);
    const float p1 = __fmul_rn(0.9997878412794807f, rad2deg), p3 = __fmul_rn(-0.3258083974640975f, rad2deg);
    const float p5 = __fmul_rn(0.1555786518463281f, rad2deg), p7 = __fmul_rn(-0.04432655554792128f, rad2deg);
    const float eps = (float)2.2204460492503131e-16;
    const float ax = fabsf(x), ay = fabsf(y);
    float a, c, c2;
    if (ax >= ay) {
        c = __fdiv_rn(ay, __fadd_rn(ax, eps));
        c2 = __fmul_rn(c, c);
        a = __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c);
    } else {
        c = __fdiv_rn(ax, __fadd_rn(ay, eps));
        c2 = __fmul_rn(c, c);
        a = __fsub_rn(90.f, __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c));
    }
    if (x < 0) a = __fsub_rn(180.f, a);
    if (y < 0) a = __fsub_rn(360.f, a);
    return a;
}

constexpr int kUploadChunk = 16;        // frames per upload/compute chunk of the host-buffer path
// K4+K5 fused: descriptor blur + IC-angle orientation + rBRIEF + scale correction, one warp per keypoint.
//   The reference blurs the WHOLE level (cv::GaussianBlur 7x7 sigma 2 REFLECT_101, orb_extractor.cc:103) and then samples 512 points
//   within radius 18.4 of every keypoint.  Both passes of the fixed-point Gaussian are integer (Q8.8 taps, one rounding at the very
//   end), so the blurred value of a pixel depends only on its 7x7 neighbourhood: blurring just the 37x37 window a keypoint can sample
//   gives the same bytes.  Per keypoint the warp
//     1. receives the un-blurred 43 x 43 neighbourhood as ONE cp.async.bulk.tensor box (64 x 43 bytes, origin on a 16-byte boundary;
//        out-of-image bytes arrive as zeros and the <= 2 rows / columns beyond the border are then filled in by REFLECT_101), while it
//        still works on the previous keypoint (two tile buffers and two mbarriers per warp);
//     2. runs the horizontal pass (dp4a, exact 16-bit sums stored as vertical pairs) and the vertical pass (dp2a, Q16.16, rounded) in its
//        private shared memory -- the arithmetic of the former whole-level kernel, on 1 369 instead of 6.4 M pixels per frame;
//     3. takes the intensity-centroid angle from the same un-blurred tile and the 256 rBRIEF comparisons from the blurred window.
//   This removes the blurred pyramid (2 x 6.4 MB per frame of HBM traffic) and the sector-granular global gathers of the descriptor.
constexpr int kDescWarps = 8;             // warps per block
constexpr int kDescBlocksPerFrame = 37;   // blockIdx.x range (x batch = a multiple of the SM count for 64 frames); warps stride over keypoints
constexpr int kFdR = 18;                  // largest |row| / |column| offset an rBRIEF sample can have (pattern radius 18.38)
constexpr int kFdWin = 2 * kFdR + 1;      // 37: blurred window
constexpr int kFdIn = kFdWin + 6;         // 43: un-blurred rows / columns it depends on
constexpr int kFdTileW = 64;              // bytes per tile row = width of the TMA box
constexpr int kFdTileBytes = 2816;        // 44 rows x 64 (43 used), a multiple of 128
constexpr int kFdHpW = 40;                // columns of the horizontal / vertical pass (37 used)
constexpr int kFdHpRows = 22;             // pair-rows of the horizontal pass (rows 0..43)
struct FdWarp {
    unsigned char tile[2][kFdTileBytes];
    unsigned hp[kFdHpRows * kFdHpW];
    unsigned char blur[kFdHpW * kFdHpW];
    unsigned long long bar[2];
    unsigned char pad[112];
};
static_assert(sizeof(FdWarp) % 128 == 0, "per-warp block keeps the TMA destinations 128-byte aligned");

template <bool kUseTma>
__global__ void __launch_bounds__(kDescWarps * 32) describe_kernel(const __grid_constant__ Geom g, const __grid_constant__ TmapSet tmaps, Images im,
                                                                   const RawKp* __restrict__ raw, int raw_stride, const int* __restrict__ counts,
                                                                   b200_keypoint_t* __restrict__ kps, unsigned char* __restrict__ descs,
                                                                   int out_stride, int frame0) {
    extern __shared__ __align__(128) unsigned char fd_smem[];
    const int frame = blockIdx.y;
    const int lane = threadIdx.x & 31;
    FdWarp& S = reinterpret_cast<FdWarp*>(fd_smem)[threadIdx.x >> 5];
    const int warp = blockIdx.x * kDescWarps + (threadIdx.x >> 5);
    const int n = counts[frame];
    constexpr int kStride = kDescBlocksPerFrame * kDescWarps;
    // this lane's 8 bit tests (x0,y0,x1,y1 as 4 int8 per word): a lane-varying constant-memory index would serialise
    // every access 32 ways, so the words are fetched once and kept in registers
    unsigned pat[8];
#pragma unroll
    for (int b = 0; b < 8; ++b) pat[b] = reinterpret_cast<const unsigned*>(c_pattern)[lane * 8 + b];
    if (kUseTma) {
        if (lane == 0) {
            mbar_init(&S.bar[0], 1);
            mbar_init(&S.bar[1], 1);
        }
        __syncwarp();
    }
    const RawKp* __restrict__ rawf = raw + (size_t)frame * raw_stride;
    // tile column of window column 0: the box starts at the 16-byte boundary at or below x - 22, so that the horizontal pass may read
    // one byte to the left of the window (the dp4a grouping of blur_h4 is anchored one byte early)
    auto issue = [&](int buf, const RawKp rk) {
        if (lane == 0) {
            mbar_expect_tx(&S.bar[buf], kFdTileW * kFdIn);
            tma_load_3d(S.tile[buf], &tmaps.m[rk.level], ((int)rk.x - 22) & ~15, (int)rk.y - 21, frame + (rk.level ? frame0 : 0), &S.bar[buf]);
        }
    };
    RawKp rk_next{};
    if (warp < n) {
        rk_next = rawf[warp];
        if (kUseTma) issue(0, rk_next);
    }
    int it = 0;
    for (int k = warp; k < n; k += kStride, ++it) {
        const RawKp rk = rk_next;
        const int cur = it & 1;
        if (k + kStride < n) {
            rk_next = rawf[k + kStride];
            if (kUseTma) issue(cur ^ 1, rk_next);  // (the buffer was released by the __syncwarp that ended the previous iteration)
        }
        const int level = rk.level;
        const LevelGeom& L = g.lv[level];
        const int kx = rk.x, ky = rk.y;
        const int x_start = kUseTma ? ((kx - 22) & ~15) : kx - 22;
        const int ox = kx - 21 - x_start;  // tile column of input column 0 (1..16)
        unsigned char* __restrict__ tile = S.tile[cur];
        if (kUseTma) {
            mbar_wait(&S.bar[cur], (unsigned)(it >> 1) & 1u);
            // REFLECT_101 for the (at most two) rows / columns of the neighbourhood that lie outside the level
            if (ky - 21 < 0 || ky + 21 >= L.h || kx - 21 < 0 || kx + 21 >= L.w) {
                for (int tr = 0; tr < kFdIn; ++tr) {
                    const int iy = ky - 21 + tr;
                    if (iy >= 0 && iy < L.h) continue;
                    const int sr = reflect101(iy, L.h) - (ky - 21);
                    if (lane < 16) reinterpret_cast<unsigned*>(tile + tr * kFdTileW)[lane] = reinterpret_cast<const unsigned*>(tile + sr * kFdTileW)[lane];
                }
                __syncwarp();
                for (int tc = ox; tc < ox + kFdIn; ++tc) {
                    const int ix = x_start + tc;
                    if (ix >= 0 && ix < L.w) continue;
                    const int sc = reflect101(ix, L.w) - x_start;
                    for (int tr = lane; tr < kFdIn; tr += 32) tile[tr * kFdTileW + tc] = tile[tr * kFdTileW + sc];
                }
                __syncwarp();
            }
        } else {
            int pitch;
            const unsigned char* img = level_ptr(im, g, level, frame, &pitch);
            for (int idx = lane; idx < kFdIn * kFdIn; idx += 32) {
                const int tr = idx / kFdIn, j = idx - tr * kFdIn;
                tile[tr * kFdTileW + ox + j] = img[(size_t)reflect101(ky - 21 + tr, L.h) * pitch + reflect101(kx - 21 + j, L.w)];
            }
            __syncwarp();
        }
        // ---- horizontal pass (exact: sum <= 65280): item = (pair-row, group of four columns), stored as vertical u16 pairs
        {
            const int bb0 = ox - 1, sh = (bb0 & 3) * 8, w0i = bb0 >> 2;
            for (int idx = lane; idx < kFdHpRows * (kFdHpW / 4); idx += 32) {
                const int pr = idx / (kFdHpW / 4), q = idx - pr * (kFdHpW / 4);
                const unsigned* r0 = reinterpret_cast<const unsigned*>(tile + (2 * pr) * kFdTileW) + w0i + q;
                const unsigned* r1 = r0 + kFdTileW / 4;
                unsigned h0[4], h1[4];
                {
                    const unsigned a0 = r0[0], a1 = r0[1], a2 = r0[2], a3 = r0[3];
                    blur_h4(__funnelshift_r(a0, a1, sh), __funnelshift_r(a1, a2, sh), __funnelshift_r(a2, a3, sh), h0);
                }
                {
                    const unsigned a0 = r1[0], a1 = r1[1], a2 = r1[2], a3 = r1[3];
                    blur_h4(__funnelshift_r(a0, a1, sh), __funnelshift_r(a1, a2, sh), __funnelshift_r(a2, a3, sh), h1);
                }
                uint4 o;
                o.x = h0[0] | (h1[0] << 16);
                o.y = h0[1] | (h1[1] << 16);
                o.z = h0[2] | (h1[2] << 16);
                o.w = h0[3] | (h1[3] << 16);
                *reinterpret_cast<uint4*>(S.hp + pr * kFdHpW + 4 * q) = o;
            }
        }
        __syncwarp();
        // ---- vertical pass: Q16.16 accumulate with dp2a on the vertical pairs, round to nearest, saturate.  item = (column, 8 rows)
        {
            constexpr unsigned E01 = 18u | (34u << 8) | (48u << 16) | (56u << 24), E23 = 48u | (34u << 8) | (18u << 16);
            constexpr unsigned O01 = (18u << 8) | (34u << 16) | (48u << 24), O23 = 56u | (48u << 8) | (34u << 16) | (18u << 24);
            for (int idx = lane; idx < kFdHpW * 5; idx += 32) {
                const int rb = idx / kFdHpW, c = idx - rb * kFdHpW;
                unsigned p[7];
#pragma unroll
                for (int t = 0; t < 7; ++t) p[t] = (4 * rb + t < kFdHpRows) ? S.hp[(4 * rb + t) * kFdHpW + c] : 0u;
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    unsigned e = __dp2a_lo(p[i], E01, 0u);
                    e = __dp2a_hi(p[i + 1], E01, e);
                    e = __dp2a_lo(p[i + 2], E23, e);
                    e = __dp2a_hi(p[i + 3], E23, e);
                    unsigned o = __dp2a_lo(p[i], O01, 0u);
                    o = __dp2a_hi(p[i + 1], O01, o);
                    o = __dp2a_lo(p[i + 2], O23, o);
                    o = __dp2a_hi(p[i + 3], O23, o);
                    S.blur[(8 * rb + 2 * i) * kFdHpW + c] = (unsigned char)min((e + 32768u) >> 16, 255u);
                    S.blur[(8 * rb + 2 * i + 1) * kFdHpW + c] = (unsigned char)min((o + 32768u) >> 16, 255u);
                }
            }
        }
        // ---- ic_angle (orb_impl.cc:68-91) on the un-blurred tile: m10 = sum u*I, m01 = sum v*I over the radius-15 disc
        int m10 = 0, m01 = 0;
        if (lane < 31) {
            const int u = lane - 15, au = abs(u);
            const unsigned char* c = tile + 21 * kFdTileW + ox + 21 + u;
            int col = 0;
#pragma unroll
            for (int v = -15; v <= 15; ++v) {
                if (au <= c_umax[v < 0 ? -v : v]) {
                    const int val = c[v * kFdTileW];
                    col += val;
                    m01 += v * val;
                }
            }
            m10 = u * col;
        }
#pragma unroll
        for (int s2 = 16; s2 > 0; s2 >>= 1) {
            m10 += __shfl_xor_sync(0xFFFFFFFFu, m10, s2);
            m01 += __shfl_xor_sync(0xFFFFFFFFu, m01, s2);
        }
        const float angle = fast_atan2_deg((float)m01, (float)m10);
        __syncwarp();  // the blurred window is complete
        // ---- compute_orb_descriptor (orb_impl.cc:93-154) on the blurred window
        const float arad = (float)((double)angle * 3.14159265358979323846 / 180.0);
        const float ca = util_cos(arad), sa = util_sin(arad);
        const unsigned char* bc = S.blur + kFdR * kFdHpW + kFdR;
        unsigned val = 0;
#pragma unroll
        for (int b = 0; b < 8; ++b) {
            const float x0 = (float)(int)(signed char)(pat[b] & 0xFF), y0 = (float)(int)(signed char)((pat[b] >> 8) & 0xFF);
            const float x1 = (float)(int)(signed char)((pat[b] >> 16) & 0xFF), y1 = (float)(int)(signed char)(pat[b] >> 24);
            int r0 = __float2int_rn(__fadd_rn(__fmul_rn(x0, sa), __fmul_rn(y0, ca)));
            int c0 = __float2int_rn(__fsub_rn(__fmul_rn(x0, ca), __fmul_rn(y0, sa)));
            int r1 = __float2int_rn(__fadd_rn(__fmul_rn(x1, sa), __fmul_rn(y1, ca)));
            int c1 = __float2int_rn(__fsub_rn(__fmul_rn(x1, ca), __fmul_rn(y1, sa)));
            // (|offset| <= 18 by construction: pattern radius 18.38, |cos|, |sin| <= 1; the clamp only guards the shared-memory access)
            r0 = max(-kFdR, min(kFdR, r0)); c0 = max(-kFdR, min(kFdR, c0));
            r1 = max(-kFdR, min(kFdR, r1)); c1 = max(-kFdR, min(kFdR, c1));
            val |= (unsigned)(bc[r0 * kFdHpW + c0] < bc[r1 * kFdHpW + c1]) << b;
        }
        const size_t o = (size_t)frame * out_stride + k;
        descs[o * 32 + lane] = (unsigned char)val;
        if (lane == 0) {
            b200_keypoint_t kp;
            float x = (float)kx, y = (float)ky;
            if (level > 0) {  // correct_keypoint_scale (orb_extractor.cc:337-345)
                x = __fmul_rn(x, L.sf);
                y = __fmul_rn(y, L.sf);
            }
            kp.x = x;
            kp.y = y;
            kp.size = L.size;
            kp.angle = angle;
            kp.response = (float)(rk.m - 1);
            kp.octave = level;
            kps[o] = kp;
        }
        __syncwarp();  // every lane is done with tile[cur], hp and blur before they are reused
    }
}

// ---------------------------------------------------------------------------------------------------------------
// host side: geometry, tables, arenas
// ---------------------------------------------------------------------------------------------------------------
static inline short sat_short_rint(float v) {
    long r = lrintf(v);
    return (short)std::min(32767L, std::max(-32768L, r));
}
static inline int floor_to_int(float v) {
    int i = (int)v;
    return i - (v < (float)i);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_tiled_fn() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &p, 12000, cudaEnableDefault, &q) == cudaSuccess
            && q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

// 3-D u8 tensor map (x, y, frame) with a 96 x 72 x 1 box; false if the buffer does not meet TMA's alignment rules
// (16-byte aligned base and strides; the kernel additionally keeps the box origin x on a 16-byte boundary)
static bool make_level_tmap(CUtensorMap* out, const void* base, int w, int h, size_t pitch, size_t fstride, int frames, int box_w = kRawPitch,
                            int box_h = kTileRows) {
    EncodeTiledFn fn = encode_tiled_fn();
    if (!fn) return false;
    if ((reinterpret_cast<unsigned long long>(base) & 15ull) || (pitch & 15) || (frames > 1 && (fstride & 15)) || w < 1 || h < 1) return false;
    const cuuint64_t dims[3] = {(cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)std::max(frames, 1)};
    const cuuint64_t strides[2] = {(cuuint64_t)pitch, (cuuint64_t)(frames > 1 ? fstride : pitch * (size_t)h + ((16 - (pitch * (size_t)h) % 16) % 16))};
    const cuuint32_t box[3] = {(cuuint32_t)box_w, (cuuint32_t)box_h, 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    return fn(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
              CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE)
           == CUDA_SUCCESS;
}

struct Extractor {
    b200_orb_params_t prm{};
    std::vector<float> mask_rects;
    cudaStream_t own_stream = nullptr, stream = nullptr, copy_stream = nullptr;
    cudaEvent_t ev[8] = {};
    std::vector<cudaEvent_t> chunk_events;
    cudaEvent_t chunk_event(int i) {
        while ((int)chunk_events.size() <= i) {
            cudaEvent_t e = nullptr;
            if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) return nullptr;
            chunk_events.push_back(e);
        }
        return chunk_events[i];
    }
    bool timing = false;
    float stage_ms[6] = {};
    // configured geometry
    int width = 0, height = 0, batch_cap = 0;
    Geom geom{};
    std::vector<float> sf;
    int n_cells = 0, raw_stride = 0;
    size_t pyr_fstride = 0, img0_pitch = 0, img0_fstride = 0;
    // device arenas
    unsigned char *d_img0 = nullptr, *d_pyr = nullptr, *d_rect_mask = nullptr, *d_user_mask = nullptr;
    CellDesc* d_cells = nullptr;
    ResizeTap* d_taps = nullptr;
    unsigned long long* d_grid = nullptr;
    RawKp* d_raw = nullptr;
    int *d_counts = nullptr, *d_level_counts = nullptr, *d_raw_corners = nullptr;
    b200_keypoint_t* d_kps = nullptr;
    unsigned char* d_descs = nullptr;
    int* h_counts = nullptr;  // pinned
    int last_batch = 0;
    const unsigned char* last_img0 = nullptr;  // level 0 of the last extract (see run())
    size_t last_pitch0 = 0, last_fstride0 = 0;
    bool rect_mask_ready = false;
    TmapSet tmaps{};           // levels >= 1 are encoded once per configuration, level 0 per call (caller's pointer)
    TmapSet tmaps_desc{};      // the same levels with the 64 x 43 box of the descriptor kernel
    bool tmaps_ok = false, last_used_tma = false;
    int tmap_frames = 0;
    // caller-owned result buffers (b200_orb_bind_outputs); when null the instance's own arenas are used
    b200_keypoint_t* out_kps = nullptr;
    unsigned char* out_descs = nullptr;
    int* out_counts = nullptr;
    int out_stride = 0;
    b200_keypoint_t* res_kps() const { return out_kps ? out_kps : d_kps; }
    unsigned char* res_descs() const { return out_kps ? out_descs : d_descs; }
    int* res_counts() const { return out_kps ? out_counts : d_counts; }
    int res_stride() const { return out_kps ? out_stride : raw_stride; }

    void free_arenas() {
        cudaFree(d_img0); cudaFree(d_pyr); cudaFree(d_rect_mask); cudaFree(d_user_mask);
        cudaFree(d_cells); cudaFree(d_taps); cudaFree(d_grid); cudaFree(d_raw);
        cudaFree(d_counts); cudaFree(d_level_counts); cudaFree(d_raw_corners); cudaFree(d_kps); cudaFree(d_descs);
        if (h_counts) cudaFreeHost(h_counts);
        d_img0 = d_pyr = d_rect_mask = d_user_mask = nullptr;
        d_cells = nullptr; d_taps = nullptr; d_grid = nullptr; d_raw = nullptr;
        d_counts = d_level_counts = d_raw_corners = nullptr; d_kps = nullptr; d_descs = nullptr; h_counts = nullptr;
        rect_mask_ready = false;
    }

    static int level_geometry(const b200_orb_params_t& prm, int w, int h, Geom& g, std::vector<float>& sf) {
        const int nl = prm.num_levels;
        sf.assign(nl, 1.0f);
        for (int l = 1; l < nl; ++l) sf[l] = prm.scale_factor * sf[l - 1];  // orb_params.cc:37-43
        g = Geom{};
        g.num_levels = nl;
        g.ini_thr = std::min(255, std::max(0, prm.ini_fast_thr));
        g.min_thr = std::min(255, std::max(0, prm.min_fast_thr));
        const unsigned min_area_sqrt = (unsigned)std::sqrt((double)prm.min_area);  // orb_extractor.cc:20
        unsigned long long off = 0;
        int grid_base = 0;
        for (int l = 0; l < nl; ++l) {
            LevelGeom& L = g.lv[l];
            if (l == 0) {
                L.w = w;
                L.h = h;
            } else {  // orb_extractor.cc:157-158
                const double scale = sf[l];
                L.w = (int)std::round(w * 1.0 / scale);
                L.h = (int)std::round(h * 1.0 / scale);
            }
            if (L.w < 1 || L.h < 1) {
                set_error("pyramid level %d of a %dx%d image is empty", l, w, h);
                return B200_ERR_INVALID;
            }
            L.pitch = round_up(L.w, 64);
            L.offset = off;
            off += round_up((unsigned long long)L.pitch * L.h, 256ull);
            L.sf = sf[l];
            L.size = (float)(unsigned)(31 * sf[l]);
            L.grid_base = grid_base;
            if (L.w > 2 * kBorder && L.h > 2 * kBorder) {
                const int span_x = L.w - 2 * kBorder, span_y = L.h - 2 * kBorder;
                const double s = (double)((float)min_area_sqrt / sf[l]);  // unsigned / float, then widened
                L.nx = (int)(unsigned)std::ceil(span_x / s);
                L.ny = (int)(unsigned)std::ceil(span_y / s);
                L.delta_x = (double)span_x / L.nx;
                L.delta_y = (double)span_y / L.ny;
                L.ncols = span_x / kCell + 1;
            } else {
                L.nx = L.ny = 0;
                L.delta_x = L.delta_y = 1.0;
                L.ncols = 1;
            }
            grid_base += L.nx * L.ny;
        }
        g.grid_cells = grid_base;
        return B200_OK;
    }

    int configure(int w, int h, int batch) {
        if (w == width && h == height && batch <= batch_cap) return B200_OK;
        B200_CUDA(cudaStreamSynchronize(stream));
        free_arenas();
        width = height = batch_cap = 0;
        int rc = level_geometry(prm, w, h, geom, sf);
        if (rc) return rc;
        const int nl = geom.num_levels;
        // FAST cells in the reference's scan order (orb_extractor.cc:199-217)
        std::vector<CellDesc> cells;
        std::vector<ResizeTap> taps;
        for (int l = 0; l < nl; ++l) {
            LevelGeom& L = geom.lv[l];
            if (L.w > 2 * kBorder && L.h > 2 * kBorder) {
                const unsigned max_bx = L.w - kBorder, max_by = L.h - kBorder;
                const unsigned ncols = (max_bx - kBorder) / kCell + 1, nrows = (max_by - kBorder) / kCell + 1;
                for (unsigned i = 0; i < nrows; ++i) {
                    const unsigned min_y = kBorder + i * kCell;
                    if (max_by - kOverlap <= min_y) continue;
                    const unsigned max_y = std::min(min_y + kCell + kOverlap, max_by);
                    for (unsigned j = 0; j < ncols; ++j) {
                        const unsigned min_x = kBorder + j * kCell;
                        if (max_bx - kOverlap <= min_x) continue;
                        const unsigned max_x = std::min(min_x + kCell + kOverlap, max_bx);
                        CellDesc c{};
                        c.level = (unsigned short)l; c.i = (unsigned short)i; c.j = (unsigned short)j;
                        c.min_x = (unsigned short)min_x; c.min_y = (unsigned short)min_y;
                        c.w = (unsigned short)(max_x - min_x); c.h = (unsigned short)(max_y - min_y);
                        cells.push_back(c);
                    }
                }
            }
            // resize taps l-1 -> l (OpenCV resize.cpp: fx clamped at the borders, rows clipped)
            if (l > 0) {
                const LevelGeom& S = geom.lv[l - 1];
                const double inv_sx = (double)L.w / S.w, inv_sy = (double)L.h / S.h;
                const double scale_x = 1. / inv_sx, scale_y = 1. / inv_sy;
                L.tab_x = (int)taps.size();
                for (int dx = 0; dx < L.w; ++dx) {
                    float fx = (float)((dx + 0.5) * scale_x - 0.5);
                    int sx = floor_to_int(fx);
                    fx -= sx;
                    if (sx < 0) { fx = 0; sx = 0; }
                    if (sx >= S.w - 1) { fx = 0; sx = S.w - 1; }
                    taps.push_back(ResizeTap{(short)sx, sat_short_rint((1.f - fx) * 2048.f), sat_short_rint(fx * 2048.f), 0});
                }
                L.tab_y = (int)taps.size();
                for (int dy = 0; dy < L.h; ++dy) {
                    float fy = (float)((dy + 0.5) * scale_y - 0.5);
                    int sy = floor_to_int(fy);
                    fy -= sy;
                    taps.push_back(ResizeTap{(short)sy, sat_short_rint((1.f - fy) * 2048.f), sat_short_rint(fy * 2048.f), 0});
                }
            }
        }
        if (geom.lv[0].w > 32767 || geom.lv[0].h > 32767) {
            set_error("image %dx%d too large", w, h);
            return B200_ERR_INVALID;
        }
        n_cells = (int)cells.size();
        raw_stride = std::max(1, geom.grid_cells);
        unsigned long long total = 0;
        for (int l = 0; l < nl; ++l) total = geom.lv[l].offset + round_up((unsigned long long)geom.lv[l].pitch * geom.lv[l].h, 256ull);
        pyr_fstride = total;
        img0_pitch = geom.lv[0].pitch;
        img0_fstride = (size_t)img0_pitch * h;

        B200_CUDA(cudaMalloc(&d_img0, img0_fstride * batch));
        B200_CUDA(cudaMalloc(&d_pyr, pyr_fstride * batch));
        B200_CUDA(cudaMalloc(&d_user_mask, img0_fstride));
        B200_CUDA(cudaMalloc(&d_cells, sizeof(CellDesc) * std::max(1, n_cells)));
        B200_CUDA(cudaMalloc(&d_taps, sizeof(ResizeTap) * std::max<size_t>(1, taps.size())));
        B200_CUDA(cudaMalloc(&d_grid, sizeof(unsigned long long) * (size_t)raw_stride * batch));
        B200_CUDA(cudaMalloc(&d_raw, sizeof(RawKp) * (size_t)raw_stride * batch));
        B200_CUDA(cudaMalloc(&d_counts, sizeof(int) * batch));
        B200_CUDA(cudaMalloc(&d_level_counts, sizeof(int) * kMaxLevels * batch));
        B200_CUDA(cudaMalloc(&d_raw_corners, sizeof(int) * batch));
        B200_CUDA(cudaMalloc(&d_kps, sizeof(b200_keypoint_t) * (size_t)raw_stride * batch));
        B200_CUDA(cudaMalloc(&d_descs, (size_t)32 * raw_stride * batch));
        B200_CUDA(cudaHostAlloc(&h_counts, sizeof(int) * (kMaxLevels + 1) * batch, cudaHostAllocDefault));
        if (n_cells) B200_CUDA(cudaMemcpyAsync(d_cells, cells.data(), sizeof(CellDesc) * n_cells, cudaMemcpyHostToDevice, stream));
        if (!taps.empty()) B200_CUDA(cudaMemcpyAsync(d_taps, taps.data(), sizeof(ResizeTap) * taps.size(), cudaMemcpyHostToDevice, stream));
        // create_rectangle_mask (orb_extractor.cc:138-151): zero set of the filled rectangles
        if (!mask_rects.empty()) {
            std::vector<unsigned char> m((size_t)img0_pitch * h, 255);
            for (size_t r = 0; r + 3 < mask_rects.size(); r += 4) {
                const unsigned x_min = (unsigned)std::round(w * mask_rects[r]), x_max = (unsigned)std::round(w * mask_rects[r + 1]);
                const unsigned y_min = (unsigned)std::round(h * mask_rects[r + 2]), y_max = (unsigned)std::round(h * mask_rects[r + 3]);
                for (unsigned y = y_min; y <= y_max && y < (unsigned)h; ++y)
                    for (unsigned x = x_min; x <= x_max && x < (unsigned)w; ++x) m[(size_t)y * img0_pitch + x] = 0;
            }
            B200_CUDA(cudaMalloc(&d_rect_mask, (size_t)img0_pitch * h));
            B200_CUDA(cudaMemcpyAsync(d_rect_mask, m.data(), m.size(), cudaMemcpyHostToDevice, stream));
            B200_CUDA(cudaStreamSynchronize(stream));
            rect_mask_ready = true;
        }
        B200_CUDA(cudaStreamSynchronize(stream));
        tmaps_ok = true;
        tmap_frames = batch;
        for (int l = 1; l < nl && tmaps_ok; ++l)
            tmaps_ok = make_level_tmap(&tmaps.m[l], d_pyr + geom.lv[l].offset, geom.lv[l].w, geom.lv[l].h, geom.lv[l].pitch, pyr_fstride, batch)
                       && make_level_tmap(&tmaps_desc.m[l], d_pyr + geom.lv[l].offset, geom.lv[l].w, geom.lv[l].h, geom.lv[l].pitch, pyr_fstride, batch,
                                          kFdTileW, kFdIn);
        width = w;
        height = h;
        batch_cap = batch;
        return B200_OK;
    }

    // Enqueue the whole extractor for `batch` frames.  frame0: first slot of the arenas / result buffers to use, so that a large
    // host batch can be processed in chunks while later chunks are still being uploaded.
    int run(const void* d_images, size_t pitch, size_t fstride, int batch, const void* d_mask, size_t mask_pitch, int frame0 = 0,
            bool record = true) {
        Images im{(const unsigned char*)d_images, pitch, fstride, d_pyr + (size_t)frame0 * pyr_fstride, pyr_fstride};
        // level 0 of frame f of this extract: last_img0 + f * last_fstride0 (the caller's buffer, or the upload staging)
        last_img0 = (const unsigned char*)d_images - (size_t)frame0 * fstride;
        last_pitch0 = pitch;
        last_fstride0 = fstride;
        const unsigned char* mask = (const unsigned char*)d_mask;
        unsigned long long mpitch = mask_pitch;
        if (!mask && rect_mask_ready) {  // orb_extractor.cc:50-64: image mask first, else rectangle mask
            mask = d_rect_mask;
            mpitch = img0_pitch;
        }
        if (out_kps && out_stride < geom.grid_cells) {
            set_error("bound output stride %d is smaller than the keypoint upper bound %d", out_stride, geom.grid_cells);
            return B200_ERR_CAPACITY;
        }
        const int nl = geom.num_levels;
        const bool tm = timing && record;
        unsigned long long* grid = d_grid + (size_t)frame0 * geom.grid_cells;
        RawKp* raw = d_raw + (size_t)frame0 * raw_stride;
        int* counts = res_counts() + frame0;
        if (tm) B200_CUDA(cudaEventRecord(ev[0], stream));
        for (int l = 1; l < nl; ++l) {
            const LevelGeom& L = geom.lv[l];
            dim3 grd(ceil_div(L.pitch / 4, 128), ceil_div(L.h, kRzRows), batch);
            resize_kernel<<<grd, 128, 0, stream>>>(geom, im, d_taps, l);
        }
        if (tm) B200_CUDA(cudaEventRecord(ev[1], stream));
        B200_CUDA(cudaMemsetAsync(grid, 0, sizeof(unsigned long long) * (size_t)std::max(1, geom.grid_cells) * batch, stream));
        B200_CUDA(cudaMemsetAsync(d_raw_corners + frame0, 0, sizeof(int) * batch, stream));
        if (n_cells) {
            // level 0 lives in the caller's buffer: encode its tensor map for this call (a host-side table fill, no GPU work)
            const bool tma = tmaps_ok && make_level_tmap(&tmaps.m[0], d_images, geom.lv[0].w, geom.lv[0].h, pitch, fstride, batch);
            if (tma) fast_cells_kernel<true><<<dim3(n_cells, batch), kFastThreads, 0, stream>>>(geom, tmaps, im, d_cells, mask, mpitch, grid, frame0,
                                                                                                   d_raw_corners + frame0);
            else fast_cells_kernel<false><<<dim3(n_cells, batch), kFastThreads, 0, stream>>>(geom, tmaps, im, d_cells, mask, mpitch, grid, frame0,
                                                                                                    d_raw_corners + frame0);
            last_used_tma = tma;
        }
        if (tm) B200_CUDA(cudaEventRecord(ev[2], stream));
        select_kernel<<<dim3(nl, batch), 256, 0, stream>>>(geom, grid, raw, raw_stride, counts, d_level_counts + (size_t)frame0 * kMaxLevels);
        if (tm) B200_CUDA(cudaEventRecord(ev[3], stream));
        if (tm) B200_CUDA(cudaEventRecord(ev[4], stream));  // (stage 3, the separate blur pass, no longer exists: the descriptor kernel blurs its own windows)
        {
            const size_t smem = sizeof(FdWarp) * kDescWarps;
            const bool tma = tmaps_ok
                             && make_level_tmap(&tmaps_desc.m[0], d_images, geom.lv[0].w, geom.lv[0].h, pitch, fstride, batch, kFdTileW, kFdIn);
            b200_keypoint_t* okps = res_kps() + (size_t)frame0 * res_stride();
            unsigned char* odesc = res_descs() + (size_t)frame0 * res_stride() * 32;
            if (tma) {
                B200_CUDA(cudaFuncSetAttribute(describe_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                describe_kernel<true><<<dim3(kDescBlocksPerFrame, batch), kDescWarps * 32, smem, stream>>>(geom, tmaps_desc, im, raw, raw_stride, counts, okps,
                                                                                                          odesc, res_stride(), frame0);
            } else {
                B200_CUDA(cudaFuncSetAttribute(describe_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                describe_kernel<false><<<dim3(kDescBlocksPerFrame, batch), kDescWarps * 32, smem, stream>>>(geom, tmaps_desc, im, raw, raw_stride, counts, okps,
                                                                                                           odesc, res_stride(), frame0);
            }
        }
        if (tm) B200_CUDA(cudaEventRecord(ev[5], stream));
        B200_CUDA(cudaGetLastError());
        last_batch = frame0 + batch;
        return B200_OK;
    }
};

// ---------------------------------------------------------------------------------------------------------------
// Per-keypoint steps between the extractor and the matchers (SURVEY 8f N2):
//   camera::perspective::undistort_keypoints  (src/stella_vslam/camera/perspective.cc:245-275) = cv::undistortPoints with
//       TermCriteria(EPS | MAX_ITER, 20, 1e-6), R = I, P = K: fixed-point iteration in double, float output
//   camera::fisheye::undistort_keypoints (camera/fisheye.cc:281-309) = cv::fisheye::undistortPoints with the default
//       TermCriteria(MAX_ITER + EPS, 10, 1e-8), R = empty, P = K, K and D as CV_32F (fisheye.cc:21-22)
//   camera::radial_division::undistort_point (camera/radial_division.cc:83-98), closed form
//   camera::base::convert_keypoints_to_bearings (camera/base.cc:158-162) with perspective / equirectangular convert_point_to_bearing
//       (perspective.cc:117-122, equirectangular.cc:42-49; fisheye.cc:156-161 and radial_division.cc:100-105 are the perspective formula)
// One thread per keypoint; this file is compiled with -fmad=false, so the double arithmetic is evaluated as written.  The model is a
// launch parameter: every thread of a launch takes the same branch.
// ---------------------------------------------------------------------------------------------------------------
// camera::*::undistort_keypoints for one keypoint: perspective (cv::undistortPointsIter, 20 iterations / 1e-6), fisheye
// (cv::fisheye::undistortPoints), radial division (closed form); identity for equirectangular
__device__ __forceinline__ void undistort_point(const CamModel& c, const b200_keypoint_t& kp, float& ux, float& uy) {
    ux = kp.x;
    uy = kp.y;
    if (c.model == 2) {
        // cv_cam_matrix_ / cv_dist_params_ are cv::Mat_<float>: OpenCV widens their float values to double
        const double fx = (float)c.fx, fy = (float)c.fy, cx = (float)c.cx, cy = (float)c.cy;
        const double k0 = (float)c.k1, k1 = (float)c.k2, k2 = (float)c.k3, k3 = (float)c.k4;
        const double pwx = ((double)kp.x - cx) / fx, pwy = ((double)kp.y - cy) / fy;
        const double kHalfPi = 3.14159265358979323846 / 2.;
        double theta_d = sqrt(pwx * pwx + pwy * pwy);
        theta_d = (-kHalfPi < theta_d) ? theta_d : -kHalfPi;  // min(max(-pi/2, theta_d), pi/2): valid up to a 180 degree FOV
        theta_d = (kHalfPi < theta_d) ? kHalfPi : theta_d;
        bool converged = false;
        double theta = theta_d, scale = 0.0;
        if (fabs(theta_d) > 1e-8) {
            for (int j = 0; j < 10; ++j) {  // Newton on theta (1 + k0 t^2 + k1 t^4 + k2 t^6 + k3 t^8) = theta_d
                const double theta2 = theta * theta, theta4 = theta2 * theta2, theta6 = theta4 * theta2, theta8 = theta6 * theta2;
                const double k0_theta2 = k0 * theta2, k1_theta4 = k1 * theta4, k2_theta6 = k2 * theta6, k3_theta8 = k3 * theta8;
                const double theta_fix = (theta * (1 + k0_theta2 + k1_theta4 + k2_theta6 + k3_theta8) - theta_d)
                                         / (1 + 3 * k0_theta2 + 5 * k1_theta4 + 7 * k2_theta6 + 9 * k3_theta8);
                theta = theta - theta_fix;
                if (fabs(theta_fix) < 1e-8) {
                    converged = true;
                    break;
                }
            }
            scale = tan(theta) / theta_d;
        } else {
            converged = true;
        }
        const bool theta_flipped = (theta_d < 0 && theta > 0) || (theta_d > 0 && theta < 0);
        if (converged && !theta_flipped) {  // P * (pu, 1) with P = K: the zero entries of K add nothing
            ux = (float)(fx * (pwx * scale) + cx);
            uy = (float)(fy * (pwy * scale) + cy);
        } else {
            ux = uy = -1000000.f;
        }
    } else if (c.model == 3) {
        const double px = ((double)kp.x - c.cx) / c.fx, py = ((double)kp.y - c.cy) / c.fy;
        const double undistortion = 1.0 + c.distortion * (px * px + py * py);
        ux = (float)(px / undistortion * c.fx + c.cx);
        uy = (float)(py / undistortion * c.fy + c.cy);
    } else if (c.model == 0) {
        const double ifx = 1. / c.fx, ify = 1. / c.fy;
        const double u = kp.x, v = kp.y;
        double x = (u - c.cx) * ifx, y = (v - c.cy) * ify;
        const double x0 = x, y0 = y;
        double error = 1.7976931348623157e308;
        for (int j = 0; j < 20 && !(error < 1e-6); ++j) {
            double r2 = x * x + y * y;
            const double icdist = 1.0 / (1 + ((c.k3 * r2 + c.k2) * r2 + c.k1) * r2);  // k[5..7] = 0: the numerator is exactly 1
            if (icdist < 0) {
                x = (u - c.cx) * ifx;
                y = (v - c.cy) * ify;
                break;
            }
            const double deltaX = 2 * c.p1 * x * y + c.p2 * (r2 + 2 * x * x);
            const double deltaY = c.p1 * (r2 + 2 * y * y) + 2 * c.p2 * x * y;
            x = (x0 - deltaX) * icdist;
            y = (y0 - deltaY) * icdist;
            r2 = x * x + y * y;
            const double r4 = r2 * r2, r6 = r4 * r2;
            const double a1 = 2 * x * y, a2 = r2 + 2 * x * x, a3 = r2 + 2 * y * y;
            const double cdist = 1 + c.k1 * r2 + c.k2 * r4 + c.k3 * r6;
            const double xd0 = x * cdist + c.p1 * a1 + c.p2 * a2, yd0 = y * cdist + c.p1 * a3 + c.p2 * a1;
            const double ex = (xd0 * c.fx + c.cx) - u, ey = (yd0 * c.fy + c.cy) - v;
            error = sqrt(ex * ex + ey * ey);
        }
        ux = (float)(c.fx * x + c.cx);
        uy = (float)(c.fy * y + c.cy);
    }
}

// undist_keypts.resize(n): default cv::KeyPoint, then pt / angle / size / octave (perspective.cc:266-272, fisheye.cc:300-306,
// base.cc:124-150); equirectangular copies the keypoints as they are
__device__ __forceinline__ b200_keypoint_t undistorted_record(const CamModel& c, const b200_keypoint_t& kp, float ux, float uy) {
    b200_keypoint_t o;
    o.x = ux;
    o.y = uy;
    o.size = kp.size;
    o.angle = kp.angle;
    o.response = (c.model == 1) ? kp.response : 0.f;
    o.octave = kp.octave;
    return o;
}

// camera::*::convert_point_to_bearing of an undistorted point
__device__ __forceinline__ void point_to_bearing(const CamModel& c, float ux, float uy, double* b) {
    if (c.model == 1) {
        const double kTwoPi = 2.0 * 3.14159265358979323846, kPi = 3.14159265358979323846;
        // cols_ / rows_ are unsigned int in the reference (camera/base.h:105-107): float / unsigned is a FLOAT division
        const double lon = ((double)__fdiv_rn(ux, (float)(unsigned)c.cols) - 0.5) * kTwoPi;
        const double lat = -((double)__fdiv_rn(uy, (float)(unsigned)c.rows) - 0.5) * kPi;
        b[0] = cos(lat) * sin(lon);
        b[1] = -sin(lat);
        b[2] = cos(lat) * cos(lon);
    } else {
        const double xn = ((double)ux - c.cx) / c.fx, yn = ((double)uy - c.cy) / c.fy;
        const double l2 = sqrt(xn * xn + yn * yn + 1.0);
        b[0] = xn / l2;
        b[1] = yn / l2;
        b[2] = 1.0 / l2;
    }
}

__global__ void __launch_bounds__(128) undistort_bearings_kernel(CamModel c, const b200_keypoint_t* __restrict__ in, int n,
                                                                 b200_keypoint_t* __restrict__ out, double* __restrict__ bearings) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const b200_keypoint_t kp = in[i];
    float ux, uy;
    undistort_point(c, kp, ux, uy);
    if (out) out[i] = undistorted_record(c, kp, ux, uy);
    if (bearings) point_to_bearing(c, ux, uy, bearings + 3 * (size_t)i);
}

// system::create_RGBD_frame after the extraction (system.cc:467-530) for frame f = blockIdx.y of the last extract: the undistorted
// keypoint and bearing of undistort_bearings_kernel, then the depth sampled at the DISTORTED keypoint, img_depth.at<float>(y, x) with the
// float coordinates truncated to int.  util::convert_to_true_depth (image_converter.cc:41-43) is convertTo(CV_32F, 1.0 / factor); only
// the sampled pixel is converted: 16UC1 -> (float)v * (float)(1 / factor), 32FC1 -> v * (float)(1 / factor), or v itself when the
// factor is 1 (convertTo then copies).  x_right = undist_x - focal_x_baseline / depth in double, rounded once to float.
struct RgbdArgs {
    CamModel cam;
    double fxb;
    float scale;                 // (float)(1.0 / depthmap_factor)
    int is_16u, copy;            // depth type; 32FC1 with factor 1
    int w, h;
    unsigned long long pitch, fstride;
    int kp_stride, cap;
};
__global__ void __launch_bounds__(128) rgbd_depths_kernel(RgbdArgs a, const b200_keypoint_t* __restrict__ kps, const int* __restrict__ counts,
                                                          const unsigned char* __restrict__ maps, b200_keypoint_t* __restrict__ undist,
                                                          double* __restrict__ bearings, float* __restrict__ depths, float* __restrict__ x_right) {
    const int f = blockIdx.y;
    const int n = min(counts[f], a.cap);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const b200_keypoint_t kp = kps[(size_t)f * a.kp_stride + i];
    float ux, uy;
    undistort_point(a.cam, kp, ux, uy);
    const size_t o = (size_t)f * a.cap + i;
    undist[o] = undistorted_record(a.cam, kp, ux, uy);
    point_to_bearing(a.cam, ux, uy, bearings + 3 * o);
    const int xi = (int)kp.x, yi = (int)kp.y;
    float depth = -1.f;  // a keypoint never lies outside the frame; the guard only keeps the read inside the map
    if (0 <= xi && xi < a.w && 0 <= yi && yi < a.h) {
        const unsigned char* row = maps + (size_t)f * a.fstride + (size_t)yi * a.pitch;
        if (a.is_16u) depth = __fmul_rn((float)reinterpret_cast<const unsigned short*>(row)[xi], a.scale);
        else {
            const float v = reinterpret_cast<const float*>(row)[xi];
            depth = a.copy ? v : __fmul_rn(v, a.scale);
        }
    }
    if (!(0.f < depth)) {  // system.cc:505-507 tests depth <= 0, which a NaN passes; here a NaN is invalid too (DESIGN.md section 8)
        depths[o] = -1.f;
        x_right[o] = -1.f;
    } else {
        depths[o] = depth;
        x_right[o] = __double2float_rn(__dsub_rn((double)ux, __ddiv_rn(a.fxb, (double)depth)));
    }
}

// util::convert_to_grayscale (src/stella_vslam/util/image_converter.cc:8-39) = cv::cvtColor(COLOR_{RGB,BGR}[A]2GRAY) for 8-bit frames:
// gray = (B 3735 + G 19235 + R 9798 + 2^14) >> 15.  Pure streaming (3 or 4 bytes in, 1 byte out per pixel): one thread converts
// four pixels from three (four) 32-bit loads into one 32-bit store; rows are independent so any pitch that is a multiple of 4 works.
template <int kChannels>
__global__ void __launch_bounds__(256) gray_kernel(const unsigned char* __restrict__ src, unsigned long long spitch, unsigned long long sframe,
                                                   unsigned char* __restrict__ dst, unsigned long long dpitch, unsigned long long dframe, int w, int h,
                                                   int rgb_order) {
    const int gx = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, f = blockIdx.z;
    const int x0 = gx * 4;
    if (x0 >= w) return;
    const unsigned char* srow = src + (size_t)f * sframe + (size_t)y * spitch;
    unsigned char* drow = dst + (size_t)f * dframe + (size_t)y * dpitch;
    const unsigned cr = rgb_order ? 9798u : 3735u, cb = rgb_order ? 3735u : 9798u;  // weight of channel 0 / channel 2
    if (x0 + 4 <= w) {
        const unsigned* p = reinterpret_cast<const unsigned*>(srow + (size_t)x0 * kChannels);
        unsigned px[4];  // channel bytes of pixel k in the low 24 bits
        if (kChannels == 4) {
            px[0] = p[0]; px[1] = p[1]; px[2] = p[2]; px[3] = p[3];  // (rows are only 4-byte aligned in general)
        } else {
            const unsigned a = p[0], b = p[1], c = p[2];
            px[0] = a;
            px[1] = __funnelshift_r(a, b, 24);
            px[2] = __funnelshift_r(b, c, 16);
            px[3] = c >> 8;
        }
        unsigned out = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const unsigned c0 = px[k] & 0xFF, c1 = (px[k] >> 8) & 0xFF, c2 = (px[k] >> 16) & 0xFF;
            out |= ((c0 * cr + c1 * 19235u + c2 * cb + (1u << 14)) >> 15) << (8 * k);
        }
        *reinterpret_cast<unsigned*>(drow + x0) = out;
    } else {
        for (int x = x0; x < w; ++x) {
            const unsigned char* q = srow + (size_t)x * kChannels;
            drow[x] = (unsigned char)((q[0] * cr + q[1] * 19235u + q[2] * cb + (1u << 14)) >> 15);
        }
    }
}

// 16 pixels per thread with 128-bit loads / stores for frames whose rows are 16-byte aligned (the usual case: 1920 x 3 = 5760 B).
template <int kChannels>
__global__ void __launch_bounds__(128) gray16_kernel(const unsigned char* __restrict__ src, unsigned long long spitch, unsigned long long sframe,
                                                     unsigned char* __restrict__ dst, unsigned long long dpitch, unsigned long long dframe, int w, int h,
                                                     int rgb_order) {
    const int gx = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, f = blockIdx.z;
    const int x0 = gx * 16;
    if (x0 >= w) return;
    const unsigned char* srow = src + (size_t)f * sframe + (size_t)y * spitch;
    unsigned char* drow = dst + (size_t)f * dframe + (size_t)y * dpitch;
    const unsigned cr = rgb_order ? 9798u : 3735u, cb = rgb_order ? 3735u : 9798u;
    if (x0 + 16 <= w) {
        unsigned wds[4 * kChannels];  // 16 pixels = 12 (16) words
        const uint4* p = reinterpret_cast<const uint4*>(srow + (size_t)x0 * kChannels);
#pragma unroll
        for (int i = 0; i < kChannels; ++i) {
            const uint4 v = p[i];
            wds[4 * i] = v.x; wds[4 * i + 1] = v.y; wds[4 * i + 2] = v.z; wds[4 * i + 3] = v.w;
        }
        unsigned out[4];
#pragma unroll
        for (int g4 = 0; g4 < 4; ++g4) {  // four pixels at a time, as in gray_kernel
            unsigned px[4];
            if (kChannels == 4) {
                px[0] = wds[4 * g4]; px[1] = wds[4 * g4 + 1]; px[2] = wds[4 * g4 + 2]; px[3] = wds[4 * g4 + 3];
            } else {
                const unsigned a = wds[3 * g4], b = wds[3 * g4 + 1], c = wds[3 * g4 + 2];
                px[0] = a;
                px[1] = __funnelshift_r(a, b, 24);
                px[2] = __funnelshift_r(b, c, 16);
                px[3] = c >> 8;
            }
            unsigned o = 0;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const unsigned c0 = px[k] & 0xFF, c1 = (px[k] >> 8) & 0xFF, c2 = (px[k] >> 16) & 0xFF;
                o |= ((c0 * cr + c1 * 19235u + c2 * cb + (1u << 14)) >> 15) << (8 * k);
            }
            out[g4] = o;
        }
        *reinterpret_cast<uint4*>(drow + x0) = make_uint4(out[0], out[1], out[2], out[3]);
    } else {
        for (int x = x0; x < w; ++x) {
            const unsigned char* q = srow + (size_t)x * kChannels;
            drow[x] = (unsigned char)((q[0] * cr + q[1] * 19235u + q[2] * cb + (1u << 14)) >> 15);
        }
    }
}

// data::frame::can_observe (src/stella_vslam/data/frame.cc:59-84) for the landmarks of the local map (tracking_module.cc:559-594):
// reproject_to_image (camera/perspective.cc:130-148, equirectangular.cc:59-73), landmark::is_inside_in_orb_scale
// (data/landmark.h:88-92), the viewing-angle test and landmark::predict_scale_level (data/landmark.cc:336-353).  Thread per landmark.
struct ObserveArgs {
    CamModel cam;
    double fxb;
    float min_x, max_x, min_y, max_y;
    double Rt[12], twc[3];
    float ray_cos_thr, log_scale_factor;
    unsigned num_levels;
};
__device__ __forceinline__ bool observe_landmark(const ObserveArgs& a, double px, double py, double pz, double nx, double ny, double nz, float min_valid_i,
                                                 float max_valid_i, double& rx, double& ry, float& xr, unsigned& lvl_out) {
    bool ok = false;
    rx = 0.0;
    ry = 0.0;
    xr = 0.f;
    lvl_out = 0;
    double qx, qy;
    float qr;
    if (reproject_to_image(a.cam, a.fxb, a.min_x, a.max_x, a.min_y, a.max_y, a.Rt, px, py, pz, qx, qy, qr)) {
        const double vx = px - a.twc[0], vy = py - a.twc[1], vz = pz - a.twc[2];
        const double dist = sqrt(vx * vx + vy * vy + vz * vz);
        const float distf = (float)dist;
        const float max_dist = __fmul_rn(1.3f, max_valid_i), min_dist = __fmul_rn((float)(1.0 / 1.3), min_valid_i);
        if (min_dist <= distf && distf <= max_dist) {
            const double ray_cos = (vx * nx + vy * ny + vz * nz) / dist;
            if (!(ray_cos < (double)a.ray_cos_thr)) {
                const float ratio = __fdiv_rn(max_valid_i, distf);
                const int lvl = (int)ceilf(__fdiv_rn(logf(ratio), a.log_scale_factor));
                const float nl = (float)a.num_levels;
                lvl_out = lvl < 0 ? 0u : ((nl <= (float)(unsigned)lvl) ? (unsigned)(nl - 1.f) : (unsigned)lvl);
                ok = true;
                rx = qx;
                ry = qy;
                xr = qr;
            }
        }
    }
    return ok;
}

__global__ void __launch_bounds__(128) can_observe_kernel(ObserveArgs a, int n, const double* __restrict__ pos_w, const double* __restrict__ mean_normal,
                                                          const float* __restrict__ min_valid, const float* __restrict__ max_valid,
                                                          unsigned char* __restrict__ observable, double* __restrict__ reproj,
                                                          float* __restrict__ x_right, unsigned* __restrict__ level) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double rx, ry;
    float xr;
    unsigned lvl_out;
    const bool ok = observe_landmark(a, pos_w[3 * (size_t)i], pos_w[3 * (size_t)i + 1], pos_w[3 * (size_t)i + 2], mean_normal[3 * (size_t)i],
                                     mean_normal[3 * (size_t)i + 1], mean_normal[3 * (size_t)i + 2], min_valid[i], max_valid[i], rx, ry, xr, lvl_out);
    observable[i] = ok ? 1 : 0;
    reproj[2 * (size_t)i] = rx;
    reproj[2 * (size_t)i + 1] = ry;
    x_right[i] = xr;
    level[i] = lvl_out;
}

// data::keyframe's `undist_keypts` blob (data/keyframe.cc:324-330): cv::KeyPoint records straight from the extractor's results
__global__ void __launch_bounds__(128) keyframe_blob_kernel(CamModel c, int undistort, const b200_keypoint_t* __restrict__ in, const int* __restrict__ n_ptr,
                                                            int cap, b200_cv_keypoint_t* __restrict__ out) {
    const int n = min(*n_ptr, cap);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const b200_keypoint_t kp = in[i];
    b200_cv_keypoint_t o;
    o.x = kp.x;
    o.y = kp.y;
    o.response = kp.response;
    if (undistort) {
        undistort_point(c, kp, o.x, o.y);
        if (c.model != 1) o.response = 0.f;
    }
    o.size = kp.size;
    o.angle = kp.angle;
    o.octave = kp.octave;
    o.class_id = -1;
    out[i] = o;
}

// ---- stage A of b200_track_local_map (track_chain.cuh): the batched forms of the two kernels above, frame = blockIdx.y ----------
__device__ __forceinline__ CamModel cam_of(const chain::TrackShared& sh) {
    return CamModel{sh.model, sh.fx, sh.fy, sh.cx, sh.cy, sh.k1, sh.k2, sh.p1, sh.p2, sh.k3, sh.cols, sh.rows, sh.k4, sh.distortion};
}

__global__ void __launch_bounds__(128) track_keypoints_kernel(chain::TrackShared sh, const chain::TrackFrameDev* __restrict__ frames) {
    const chain::TrackFrameDev& F = frames[blockIdx.y];
    const int n = min(*F.n_kp, F.kp_cap);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) {
        F.status[0] = n;
        F.status[1] = ((F.kp_x_right || F.kp_landmark) && F.n_kp_in != n) ? 1 : 0;
        if (F.count_out) *F.count_out = n;
    }
    if (i >= n) return;
    const b200_keypoint_t kp = F.kps[i];
    float ux, uy;
    undistort_point(cam_of(sh), kp, ux, uy);
    b200_keypoint_t o;
    o.x = ux;
    o.y = uy;
    o.size = kp.size;
    o.angle = kp.angle;
    o.response = (sh.model == 1) ? kp.response : 0.f;
    o.octave = kp.octave;
    F.undist[i] = o;
    if (F.bearings) point_to_bearing(cam_of(sh), ux, uy, F.bearings + 3 * (size_t)i);
    F.t_x[i] = ux;
    F.t_y[i] = uy;
    F.t_octave[i] = (unsigned char)kp.octave;
    if (F.t_angle) F.t_angle[i] = kp.angle;
    unsigned char occ = 0;
    if (F.kp_landmark && i < F.n_kp_in) {  // `lm && lm->has_observation()` (projection.cc:50-53)
        const int l = F.kp_landmark[i];
        occ = (l >= 0 && l < F.n_lm && (!F.lm_has_obs || F.lm_has_obs[l])) ? 1 : 0;
    }
    F.occupied[i] = occ;
}

__global__ void __launch_bounds__(128) track_landmarks_kernel(chain::TrackShared sh, const chain::TrackFrameDev* __restrict__ frames) {
    const chain::TrackFrameDev& F = frames[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= F.n_lm) return;
    ObserveArgs a;
    a.cam = cam_of(sh);
    a.fxb = sh.fxb;
    a.min_x = sh.min_x; a.max_x = sh.max_x; a.min_y = sh.min_y; a.max_y = sh.max_y;
#pragma unroll
    for (int k = 0; k < 12; ++k) a.Rt[k] = F.Rt[k];
#pragma unroll
    for (int k = 0; k < 3; ++k) a.twc[k] = F.twc[k];
    a.ray_cos_thr = sh.ray_cos_thr;
    a.log_scale_factor = sh.log_scale_factor;
    a.num_levels = sh.num_levels;
    double rx, ry;
    float xr;
    unsigned lvl;
    bool ok = !(F.lm_skip && F.lm_skip[i]);  // tracking_module.cc:561-586: skipped before can_observe
    if (ok)
        ok = observe_landmark(a, F.pos_w[3 * (size_t)i], F.pos_w[3 * (size_t)i + 1], F.pos_w[3 * (size_t)i + 2], F.mean_normal[3 * (size_t)i],
                              F.mean_normal[3 * (size_t)i + 1], F.mean_normal[3 * (size_t)i + 2], F.min_d[i], F.max_d[i], rx, ry, xr, lvl);
    else {
        rx = ry = 0.0;
        xr = 0.f;
        lvl = 0;
    }
    F.observable[i] = ok ? 1 : 0;
    // the query of projection::match_frame_and_landmarks (projection.cc:31-38): float reprojection, octave window, scaled margin
    F.q_x[i] = (float)rx;
    F.q_y[i] = (float)ry;
    F.q_xr[i] = xr;
    F.q_margin[i] = __fmul_rn(sh.margin, sh.scale_factors[lvl]);
    F.q_lo[i] = (signed char)max(0, (int)lvl - 1);
    F.q_hi[i] = (signed char)min((int)sh.num_levels - 1, (int)lvl + 1);
    F.q_valid[i] = (unsigned char)((ok ? 1 : 0) | ((!F.lm_has_obs || F.lm_has_obs[i]) ? 2 : 0));
}

// ---- stage A of b200_motion_based_track: the query of projection::match_current_and_last_frames (projection.cc:95-160) for every entry
// of the last-frame table, frame = blockIdx.y.  The direction test runs in every thread (a few fp64 operations, -fmad=false as in the
// reference's uncontracted Eigen products).
__global__ void __launch_bounds__(128) motion_queries_kernel(chain::TrackShared sh, const chain::TrackFrameDev* __restrict__ frames) {
    const chain::TrackFrameDev& F = frames[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= F.n_lm) return;
    bool forward = false, backward = false;
    if (!sh.monocular) {  // :98-116: trans_wc = -rot_cw^T trans_cw, trans_lc = rot_lw trans_wc + trans_lw; only its z matters
        double tw[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) tw[r] = (-F.Rt[r]) * F.Rt[9] + (-F.Rt[3 + r]) * F.Rt[10] + (-F.Rt[6 + r]) * F.Rt[11];
        const double* L = F.last_Rt;
        const double z = L[6] * tw[0] + L[7] * tw[1] + L[8] * tw[2] + L[11];
        forward = z > sh.true_baseline;
        backward = -z > sh.true_baseline;
    }
    double qx = 0.0, qy = 0.0;
    float qr = 0.f;
    const bool ok = reproject_to_image(cam_of(sh), sh.fxb, sh.min_x, sh.max_x, sh.min_y, sh.max_y, F.Rt, F.pos_w[3 * (size_t)i],
                                       F.pos_w[3 * (size_t)i + 1], F.pos_w[3 * (size_t)i + 2], qx, qy, qr);
    const int lvl = F.lm_octave[i];  // < num_levels (checked by the caller)
    int lo = max(0, lvl - 1), hi = min((int)sh.num_levels - 1, lvl + 1);
    if (forward) lo = lvl;
    else if (backward) hi = lvl;
    F.q_x[i] = (float)qx;
    F.q_y[i] = (float)qy;
    F.q_xr[i] = qr;
    F.q_margin[i] = __fmul_rn(sh.margin, sh.scale_factors[lvl]);
    F.q_lo[i] = (signed char)lo;
    F.q_hi[i] = (signed char)hi;
    F.q_valid[i] = (unsigned char)((ok ? 1 : 0) | ((!F.lm_has_obs || F.lm_has_obs[i]) ? 2 : 0));
}

}  // namespace orb

namespace chain {
int track_stage_a(cudaStream_t st, const TrackShared& sh, const TrackFrameDev* d_frames, int n_frames, int max_kp, int max_lm) {
    if (max_kp > 0) orb::track_keypoints_kernel<<<dim3(ceil_div(max_kp, 128), n_frames), 128, 0, st>>>(sh, d_frames);
    if (max_lm > 0) orb::track_landmarks_kernel<<<dim3(ceil_div(max_lm, 128), n_frames), 128, 0, st>>>(sh, d_frames);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

int robust_stage_a(cudaStream_t st, const TrackShared& sh, const TrackFrameDev* d_frames, int n_frames, int max_kp) {
    if (max_kp > 0) orb::track_keypoints_kernel<<<dim3(ceil_div(max_kp, 128), n_frames), 128, 0, st>>>(sh, d_frames);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

int motion_stage_a(cudaStream_t st, const TrackShared& sh, const TrackFrameDev* d_frames, int n_frames, int max_kp, int max_lm) {
    if (max_kp > 0) orb::track_keypoints_kernel<<<dim3(ceil_div(max_kp, 128), n_frames), 128, 0, st>>>(sh, d_frames);
    if (max_lm > 0) orb::motion_queries_kernel<<<dim3(ceil_div(max_lm, 128), n_frames), 128, 0, st>>>(sh, d_frames);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}
}  // namespace chain
}  // namespace b200

using b200::orb::Extractor;

struct b200_orb_s {
    Extractor ex;
};

extern "C" {

void b200_orb_default_params(b200_orb_params_t* p) {
    if (!p) return;
    std::memset(p, 0, sizeof(*p));
    p->scale_factor = 1.2f;  // orb_params.cc:9-10
    p->num_levels = 8;
    p->ini_fast_thr = 20;
    p->min_fast_thr = 7;
    p->min_area = 800;       // system.cc:95
    p->max_batch = 1;
}

int b200_orb_create(const b200_orb_params_t* p, b200_orb_t* out) {
    if (!p || !out) {
        b200::set_error("b200_orb_create: null argument");
        return B200_ERR_INVALID;
    }
    if (p->num_levels < 1 || p->num_levels > b200::orb::kMaxLevels || !(p->scale_factor > 1.0f) || p->min_area < 1
        || p->n_mask_rects < 0 || (p->n_mask_rects > 0 && !p->mask_rects)) {
        b200::set_error("b200_orb_create: invalid parameters (levels %d, scale %f, min_area %u)", p->num_levels, p->scale_factor, p->min_area);
        return B200_ERR_INVALID;
    }
    int rc = b200::require_device(p->device);
    if (rc) return rc;
    b200_orb_s* h = new (std::nothrow) b200_orb_s();
    if (!h) return B200_ERR_INVALID;
    h->ex.prm = *p;
    h->ex.prm.mask_rects = nullptr;
    if (p->n_mask_rects > 0) h->ex.mask_rects.assign(p->mask_rects, p->mask_rects + 4 * (size_t)p->n_mask_rects);
    cudaError_t e = cudaStreamCreateWithFlags(&h->ex.own_stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&h->ex.copy_stream, cudaStreamNonBlocking);
    h->ex.stream = h->ex.own_stream;
    for (int i = 0; i < 8 && e == cudaSuccess; ++i) e = cudaEventCreate(&h->ex.ev[i]);
    if (e != cudaSuccess) {
        delete h;
        return b200::cuda_fail(e, "stream/event creation", __FILE__, __LINE__);
    }
    *out = h;
    return B200_OK;
}

int b200_orb_destroy(b200_orb_t h) {
    if (!h) return B200_OK;
    cudaSetDevice(h->ex.prm.device);
    cudaStreamSynchronize(h->ex.stream);
    h->ex.free_arenas();
    for (auto& e : h->ex.ev)
        if (e) cudaEventDestroy(e);
    for (auto& ce : h->ex.chunk_events) cudaEventDestroy(ce);
    if (h->ex.copy_stream) cudaStreamDestroy(h->ex.copy_stream);
    if (h->ex.own_stream) cudaStreamDestroy(h->ex.own_stream);
    delete h;
    return B200_OK;
}

int b200_orb_max_keypoints(b200_orb_t h, int width, int height) {
    if (!h || width <= 0 || height <= 0) return B200_ERR_INVALID;
    b200::orb::Geom g;
    std::vector<float> sf;
    int rc = Extractor::level_geometry(h->ex.prm, width, height, g, sf);
    if (rc) return rc;
    return g.grid_cells;
}

int b200_orb_extract_device(b200_orb_t h, const void* d_images, int width, int height, size_t pitch, size_t frame_stride, int batch,
                            const void* d_mask, size_t mask_pitch) {
    B200_RANGE("b200:orb:extract_device");
    if (!h) return B200_ERR_INVALID;
    if (width == 0 || height == 0 || batch == 0) {  // orb_extractor.cc:30-32: empty image -> silent return
        h->ex.last_batch = 0;
        return B200_OK;
    }
    if (!d_images || width < 0 || height < 0 || batch < 0 || pitch < (size_t)width || (batch > 1 && frame_stride < pitch * (size_t)height)) {
        b200::set_error("b200_orb_extract_device: invalid image arguments");
        return B200_ERR_INVALID;
    }
    B200_CUDA(cudaSetDevice(h->ex.prm.device));
    int rc = h->ex.configure(width, height, std::max(batch, h->ex.prm.max_batch));
    if (rc) return rc;
    return h->ex.run(d_images, pitch, frame_stride, batch, d_mask, mask_pitch);
}

int b200_orb_fetch(b200_orb_t h, b200_keypoint_t* kps, uint8_t* descs, int cap, int32_t* counts) {
    if (!h) return B200_ERR_INVALID;
    Extractor& ex = h->ex;
    if (ex.last_batch == 0) return B200_OK;
    if (!counts || cap < 0) return B200_ERR_INVALID;
    B200_CUDA(cudaSetDevice(ex.prm.device));
    const int B = ex.last_batch;
    // counts are not known on the host yet: copy min(cap, stride) records per frame with two strided copies
    const size_t m = (size_t)std::min(cap, ex.res_stride());
    B200_CUDA(cudaMemcpyAsync(ex.h_counts, ex.res_counts(), sizeof(int) * B, cudaMemcpyDeviceToHost, ex.stream));
    if (m > 0 && kps)
        B200_CUDA(cudaMemcpy2DAsync(kps, sizeof(b200_keypoint_t) * (size_t)cap, ex.res_kps(), sizeof(b200_keypoint_t) * (size_t)ex.res_stride(),
                                    sizeof(b200_keypoint_t) * m, B, cudaMemcpyDeviceToHost, ex.stream));
    if (m > 0 && descs)
        B200_CUDA(cudaMemcpy2DAsync(descs, (size_t)32 * cap, ex.res_descs(), (size_t)32 * ex.res_stride(), (size_t)32 * m, B, cudaMemcpyDeviceToHost,
                                    ex.stream));
    B200_CUDA(cudaStreamSynchronize(ex.stream));
    int rc = B200_OK;
    for (int f = 0; f < B; ++f) {
        counts[f] = ex.h_counts[f];
        if (ex.h_counts[f] > cap) {
            b200::set_error("frame %d has %d keypoints but the caller's capacity is %d", f, ex.h_counts[f], cap);
            rc = B200_ERR_CAPACITY;
        }
    }
    if (ex.timing) {
        for (int st = 0; st < 5; ++st) cudaEventElapsedTime(&ex.stage_ms[st], ex.ev[st], ex.ev[st + 1]);
        cudaEventElapsedTime(&ex.stage_ms[5], ex.ev[0], ex.ev[5]);
    }
    return rc;
}

int b200_orb_set_stream(b200_orb_t h, void* stream, int use_own) {
    if (!h) return B200_ERR_INVALID;
    B200_CUDA(cudaStreamSynchronize(h->ex.stream));
    h->ex.stream = use_own ? h->ex.own_stream : (cudaStream_t)stream;
    return B200_OK;
}

int b200_orb_bind_outputs(b200_orb_t h, void* d_kps, void* d_descs, void* d_counts, int stride_kps) {
    if (!h) return B200_ERR_INVALID;
    if (!d_kps) {  // unbind
        h->ex.out_kps = nullptr;
        h->ex.out_descs = nullptr;
        h->ex.out_counts = nullptr;
        h->ex.out_stride = 0;
        return B200_OK;
    }
    if (!d_descs || !d_counts || stride_kps <= 0) {
        b200::set_error("b200_orb_bind_outputs: all three buffers and a positive stride are required");
        return B200_ERR_INVALID;
    }
    h->ex.out_kps = (b200_keypoint_t*)d_kps;
    h->ex.out_descs = (unsigned char*)d_descs;
    h->ex.out_counts = (int*)d_counts;
    h->ex.out_stride = stride_kps;
    return B200_OK;
}

int b200_orb_reserve(b200_orb_t h, int width, int height, int batch) {
    if (!h || width <= 0 || height <= 0 || batch <= 0) return B200_ERR_INVALID;
    B200_CUDA(cudaSetDevice(h->ex.prm.device));
    return h->ex.configure(width, height, std::max(batch, h->ex.prm.max_batch));
}

int b200_orb_extract(b200_orb_t h, const uint8_t* images, int width, int height, size_t pitch, size_t frame_stride, int batch,
                     const uint8_t* mask, size_t mask_pitch, b200_keypoint_t* kps, uint8_t* descs, int cap, int32_t* counts) {
    B200_RANGE("b200:orb:extract");
    if (!h) return B200_ERR_INVALID;
    if (width == 0 || height == 0 || batch == 0) {
        h->ex.last_batch = 0;
        return B200_OK;
    }
    if (!images || width < 0 || height < 0 || batch < 0 || pitch < (size_t)width) {
        b200::set_error("b200_orb_extract: invalid image arguments");
        return B200_ERR_INVALID;
    }
    Extractor& ex = h->ex;
    B200_CUDA(cudaSetDevice(ex.prm.device));
    int rc = ex.configure(width, height, std::max(batch, ex.prm.max_batch));
    if (rc) return rc;
    const unsigned char* d_mask = nullptr;
    if (mask) {
        B200_CUDA(cudaMemcpy2DAsync(ex.d_user_mask, ex.img0_pitch, mask, mask_pitch, width, height, cudaMemcpyHostToDevice, ex.stream));
        d_mask = ex.d_user_mask;
    }
    // Chunked pipeline: the upload of chunk c+1 (copy stream) overlaps the kernels of chunk c (compute stream).
    const int chunk = batch > 2 * b200::orb::kUploadChunk ? b200::orb::kUploadChunk : batch;
    const bool contiguous = frame_stride == pitch * (size_t)height;
    int n_ev = 0;
    for (int f0 = 0; f0 < batch; f0 += chunk) {
        const int nb = std::min(chunk, batch - f0);
        cudaStream_t cs = (chunk < batch) ? ex.copy_stream : ex.stream;
        if (nb == 1 || contiguous) {  // one tall 2-D copy
            B200_CUDA(cudaMemcpy2DAsync(ex.d_img0 + (size_t)f0 * ex.img0_fstride, ex.img0_pitch, images + (size_t)f0 * frame_stride, pitch, width,
                                        (size_t)height * nb, cudaMemcpyHostToDevice, cs));
        } else {
            for (int f = f0; f < f0 + nb; ++f)
                B200_CUDA(cudaMemcpy2DAsync(ex.d_img0 + (size_t)f * ex.img0_fstride, ex.img0_pitch, images + (size_t)f * frame_stride, pitch, width,
                                            height, cudaMemcpyHostToDevice, cs));
        }
        if (cs != ex.stream) {
            cudaEvent_t e = ex.chunk_event(n_ev++);
            if (!e) return b200::cuda_fail(cudaErrorMemoryAllocation, "chunk event", __FILE__, __LINE__);
            B200_CUDA(cudaEventRecord(e, cs));
            B200_CUDA(cudaStreamWaitEvent(ex.stream, e, 0));
        }
        rc = ex.run(ex.d_img0 + (size_t)f0 * ex.img0_fstride, ex.img0_pitch, ex.img0_fstride, nb, d_mask, ex.img0_pitch, f0, chunk == batch);
        if (rc) return rc;
    }
    return b200_orb_fetch(h, kps, descs, cap, counts);
}

int b200_orb_device_results(b200_orb_t h, const b200_keypoint_t** d_kps, const uint8_t** d_descs, const int32_t** d_counts, int* stride_kps) {
    if (!h) return B200_ERR_INVALID;
    if (d_kps) *d_kps = h->ex.res_kps();
    if (d_descs) *d_descs = h->ex.res_descs();
    if (d_counts) *d_counts = h->ex.res_counts();
    if (stride_kps) *stride_kps = h->ex.res_stride();
    return B200_OK;
}

int b200_orb_sync(b200_orb_t h) {
    if (!h) return B200_ERR_INVALID;
    B200_CUDA(cudaStreamSynchronize(h->ex.stream));
    if (h->ex.timing && h->ex.last_batch > 0) {
        for (int s = 0; s < 5; ++s) cudaEventElapsedTime(&h->ex.stage_ms[s], h->ex.ev[s], h->ex.ev[s + 1]);
        cudaEventElapsedTime(&h->ex.stage_ms[5], h->ex.ev[0], h->ex.ev[5]);
    }
    return B200_OK;
}

int b200_orb_level_info(b200_orb_t h, int level, int* width, int* height, size_t* pitch, float* scale_factor) {
    if (!h || h->ex.width == 0 || level < 0 || level >= h->ex.geom.num_levels) return B200_ERR_INVALID;
    const auto& L = h->ex.geom.lv[level];
    if (width) *width = L.w;
    if (height) *height = L.h;
    if (pitch) *pitch = (size_t)L.pitch;
    if (scale_factor) *scale_factor = L.sf;
    return B200_OK;
}

int b200_orb_pyramid_level_device(b200_orb_t h, int frame, int level, const uint8_t** d_ptr) {
    if (!h || !d_ptr || h->ex.width == 0 || level < 1 || level >= h->ex.geom.num_levels || frame < 0 || frame >= h->ex.last_batch) {
        b200::set_error("b200_orb_pyramid_level_device: bad frame/level (level 0 aliases the caller's image)");
        return B200_ERR_INVALID;
    }
    *d_ptr = h->ex.d_pyr + (size_t)frame * h->ex.pyr_fstride + h->ex.geom.lv[level].offset;
    return B200_OK;
}

int b200_orb_pyramid_level_view(b200_orb_t h, int frame, int level, const uint8_t** d_ptr, size_t* pitch, int* width, int* height) {
    if (!h || !d_ptr || h->ex.width == 0 || level < 0 || level >= h->ex.geom.num_levels || frame < 0 || frame >= h->ex.last_batch) {
        b200::set_error("b200_orb_pyramid_level_view: bad frame/level");
        return B200_ERR_INVALID;
    }
    const auto& L = h->ex.geom.lv[level];
    if (level == 0) {
        if (!h->ex.last_img0) return B200_ERR_INVALID;
        *d_ptr = h->ex.last_img0 + (size_t)frame * h->ex.last_fstride0;
        if (pitch) *pitch = h->ex.last_pitch0;
    } else {
        *d_ptr = h->ex.d_pyr + (size_t)frame * h->ex.pyr_fstride + L.offset;
        if (pitch) *pitch = (size_t)L.pitch;
    }
    if (width) *width = L.w;
    if (height) *height = L.h;
    return B200_OK;
}

int b200_orb_pyramid_level_host(b200_orb_t h, int frame, int level, uint8_t* dst, size_t dst_pitch) {
    const uint8_t* d = nullptr;
    int rc = b200_orb_pyramid_level_device(h, frame, level, &d);
    if (rc) return rc;
    const auto& L = h->ex.geom.lv[level];
    if (!dst || dst_pitch < (size_t)L.w) return B200_ERR_INVALID;
    B200_CUDA(cudaMemcpy2DAsync(dst, dst_pitch, d, L.pitch, L.w, L.h, cudaMemcpyDeviceToHost, h->ex.stream));
    B200_CUDA(cudaStreamSynchronize(h->ex.stream));
    return B200_OK;
}

int b200_keypoints_undistort(b200_orb_t h, const b200_camera_intrinsics_t* cam, const b200_keypoint_t* keypts, int n, b200_keypoint_t* undist_keypts,
                             double* bearings) {
    if (!h || !cam || n < 0 || !b200::chain::camera_valid(*cam)) return B200_ERR_INVALID;
    if (n == 0) return B200_OK;  // cv::undistortPoints does not accept an empty input (perspective.cc:246-250, fisheye.cc:282-286)
    if (!keypts || (!undist_keypts && !bearings)) return B200_ERR_INVALID;
    Extractor& ex = h->ex;
    B200_CUDA(cudaSetDevice(ex.prm.device));
    const size_t kb = sizeof(b200_keypoint_t) * (size_t)n, bb = sizeof(double) * 3 * (size_t)n;
    unsigned char* d = nullptr;
    B200_CUDA(cudaMallocAsync((void**)&d, 2 * kb + bb + 512, ex.stream));
    b200_keypoint_t* d_in = reinterpret_cast<b200_keypoint_t*>(d);
    b200_keypoint_t* d_out = reinterpret_cast<b200_keypoint_t*>(d + b200::round_up(kb, (size_t)256));
    double* d_b = reinterpret_cast<double*>(d + 2 * b200::round_up(kb, (size_t)256));
    cudaError_t e = cudaMemcpyAsync(d_in, keypts, kb, cudaMemcpyHostToDevice, ex.stream);
    if (e == cudaSuccess) {
        const b200::orb::CamModel c = b200::orb::cam_model(*cam);
        b200::orb::undistort_bearings_kernel<<<b200::ceil_div(n, 128), 128, 0, ex.stream>>>(c, d_in, n, undist_keypts ? d_out : nullptr,
                                                                                         bearings ? d_b : nullptr);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess && undist_keypts) e = cudaMemcpyAsync(undist_keypts, d_out, kb, cudaMemcpyDeviceToHost, ex.stream);
    if (e == cudaSuccess && bearings) e = cudaMemcpyAsync(bearings, d_b, bb, cudaMemcpyDeviceToHost, ex.stream);
    cudaFreeAsync(d, ex.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ex.stream);
    if (e != cudaSuccess) return b200::cuda_fail(e, "b200_keypoints_undistort", __FILE__, __LINE__);
    return B200_OK;
}

int b200_frame_can_observe(b200_orb_t h, const b200_camera_intrinsics_t* cam, double focal_x_baseline, const float* img_bounds,
                           const double* pose_cw, int n, const double* pos_w, const double* mean_normal, const float* min_valid_dist,
                           const float* max_valid_dist, float ray_cos_thr, unsigned num_levels, float log_scale_factor, uint8_t* observable,
                           double* reproj, float* x_right, uint32_t* pred_scale_level) {
    if (!h || !cam || !pose_cw || n < 0 || !b200::chain::camera_valid(*cam) || (cam->model != 1 && !img_bounds)) return B200_ERR_INVALID;
    if (n == 0) return B200_OK;
    if (!pos_w || !mean_normal || !min_valid_dist || !max_valid_dist || !observable || !reproj || !x_right || !pred_scale_level) return B200_ERR_INVALID;
    Extractor& ex = h->ex;
    B200_CUDA(cudaSetDevice(ex.prm.device));
    b200::orb::ObserveArgs a{};
    a.cam = b200::orb::cam_model(*cam);
    a.fxb = focal_x_baseline;
    if (img_bounds) { a.min_x = img_bounds[0]; a.max_x = img_bounds[1]; a.min_y = img_bounds[2]; a.max_y = img_bounds[3]; }
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) a.Rt[3 * r + c] = pose_cw[4 * r + c];
        a.Rt[9 + r] = pose_cw[4 * r + 3];
    }
    for (int r = 0; r < 3; ++r)  // trans_wc_ = -rot_cw^T trans_cw (data/frame.cc: update_pose_params)
        a.twc[r] = -(a.Rt[r] * a.Rt[9] + a.Rt[3 + r] * a.Rt[10] + a.Rt[6 + r] * a.Rt[11]);
    a.ray_cos_thr = ray_cos_thr;
    a.log_scale_factor = log_scale_factor;
    a.num_levels = num_levels;
    const size_t N = (size_t)n;
    b200::Layout L;
    const size_t o_p = L.take(24 * N), o_n = L.take(24 * N), o_lo = L.take(4 * N), o_hi = L.take(4 * N);
    const size_t o_ok = L.take(N), o_rp = L.take(16 * N), o_xr = L.take(4 * N), o_lv = L.take(4 * N);
    unsigned char* d = nullptr;
    B200_CUDA(cudaMallocAsync((void**)&d, L.end, ex.stream));
    cudaStream_t st = ex.stream;
    cudaError_t e = cudaMemcpyAsync(d + o_p, pos_w, 24 * N, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d + o_n, mean_normal, 24 * N, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d + o_lo, min_valid_dist, 4 * N, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d + o_hi, max_valid_dist, 4 * N, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) {
        b200::orb::can_observe_kernel<<<b200::ceil_div(n, 128), 128, 0, st>>>(a, n, (const double*)(d + o_p), (const double*)(d + o_n), (const float*)(d + o_lo),
                                                                          (const float*)(d + o_hi), d + o_ok, (double*)(d + o_rp), (float*)(d + o_xr),
                                                                          (unsigned*)(d + o_lv));
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(observable, d + o_ok, N, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(reproj, d + o_rp, 16 * N, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(x_right, d + o_xr, 4 * N, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(pred_scale_level, d + o_lv, 4 * N, cudaMemcpyDeviceToHost, st);
    cudaFreeAsync(d, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return b200::cuda_fail(e, "b200_frame_can_observe", __FILE__, __LINE__);
    return B200_OK;
}

int b200_convert_to_grayscale_device(b200_orb_t h, const void* d_src, int width, int height, size_t src_pitch, size_t src_frame_stride, int channels,
                                     int rgb_order, void* d_gray, size_t gray_pitch, size_t gray_frame_stride, int batch) {
    if (!h || !d_src || !d_gray || width <= 0 || height <= 0 || batch <= 0 || (channels != 3 && channels != 4)
        || src_pitch < (size_t)width * channels || gray_pitch < (size_t)width || (src_pitch & 3) || (gray_pitch & 3)
        || ((uintptr_t)d_src & 15) || ((uintptr_t)d_gray & 3) || (src_frame_stride & 15) || (gray_frame_stride & 3)) {
        b200::set_error("b200_convert_to_grayscale_device: 3 or 4 channels, pitches multiples of 4, source frames 16-byte aligned");
        return B200_ERR_INVALID;
    }
    Extractor& ex = h->ex;
    B200_CUDA(cudaSetDevice(ex.prm.device));
    if (!(src_pitch & 15) && !(gray_pitch & 15) && !((uintptr_t)d_gray & 15) && !(gray_frame_stride & 15)) {  // 128-bit path
        const dim3 grid16(b200::ceil_div(b200::ceil_div(width, 16), 128), height, batch);
        if (channels == 4)
            b200::orb::gray16_kernel<4><<<grid16, 128, 0, ex.stream>>>((const unsigned char*)d_src, src_pitch, src_frame_stride, (unsigned char*)d_gray,
                                                                     gray_pitch, gray_frame_stride, width, height, rgb_order);
        else
            b200::orb::gray16_kernel<3><<<grid16, 128, 0, ex.stream>>>((const unsigned char*)d_src, src_pitch, src_frame_stride, (unsigned char*)d_gray,
                                                                     gray_pitch, gray_frame_stride, width, height, rgb_order);
        B200_CUDA(cudaGetLastError());
        return B200_OK;
    }
    const dim3 grid(b200::ceil_div(b200::ceil_div(width, 4), 256), height, batch);
    if (channels == 4)
        b200::orb::gray_kernel<4><<<grid, 256, 0, ex.stream>>>((const unsigned char*)d_src, src_pitch, src_frame_stride, (unsigned char*)d_gray, gray_pitch,
                                                             gray_frame_stride, width, height, rgb_order);
    else
        b200::orb::gray_kernel<3><<<grid, 256, 0, ex.stream>>>((const unsigned char*)d_src, src_pitch, src_frame_stride, (unsigned char*)d_gray, gray_pitch,
                                                             gray_frame_stride, width, height, rgb_order);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

int b200_convert_to_grayscale(b200_orb_t h, const uint8_t* src, int width, int height, size_t src_pitch, int channels, int rgb_order, uint8_t* gray,
                              size_t gray_pitch) {
    if (!h || !src || !gray || width <= 0 || height <= 0 || (channels != 3 && channels != 4) || src_pitch < (size_t)width * channels
        || gray_pitch < (size_t)width)
        return B200_ERR_INVALID;
    Extractor& ex = h->ex;
    B200_CUDA(cudaSetDevice(ex.prm.device));
    const size_t sp = b200::round_up((size_t)width * channels, (size_t)16), gp = b200::round_up((size_t)width, (size_t)16);
    unsigned char* d = nullptr;
    B200_CUDA(cudaMallocAsync((void**)&d, (sp + gp) * (size_t)height + 256, ex.stream));
    unsigned char* d_gray = d + b200::round_up(sp * (size_t)height, (size_t)256);
    cudaError_t e = cudaMemcpy2DAsync(d, sp, src, src_pitch, (size_t)width * channels, height, cudaMemcpyHostToDevice, ex.stream);
    int rc = B200_OK;
    if (e == cudaSuccess) rc = b200_convert_to_grayscale_device(h, d, width, height, sp, 0, channels, rgb_order, d_gray, gp, 0, 1);
    if (e == cudaSuccess && rc == B200_OK) e = cudaMemcpy2DAsync(gray, gray_pitch, d_gray, gp, width, height, cudaMemcpyDeviceToHost, ex.stream);
    cudaFreeAsync(d, ex.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ex.stream);
    if (e != cudaSuccess) return b200::cuda_fail(e, "b200_convert_to_grayscale", __FILE__, __LINE__);
    return rc;
}

int b200_orb_enable_timing(b200_orb_t h, int enable) {
    if (!h) return B200_ERR_INVALID;
    h->ex.timing = enable != 0;
    return B200_OK;
}

int b200_orb_export_keyframe_blobs(b200_orb_t h, int frame, const b200_camera_intrinsics_t* cam, b200_cv_keypoint_t* keypts_blob, uint8_t* desc_blob,
                                   int cap, int32_t* n) {
    if (!h || !n || cap < 0 || (cap > 0 && (!keypts_blob || !desc_blob)) || (cam && !b200::chain::camera_valid(*cam))) return B200_ERR_INVALID;
    Extractor& ex = h->ex;
    if (ex.width == 0 || frame < 0 || frame >= ex.last_batch) {
        b200::set_error("b200_orb_export_keyframe_blobs: frame %d is not part of the last extract", frame);
        return B200_ERR_INVALID;
    }
    B200_CUDA(cudaSetDevice(ex.prm.device));
    const int stride = ex.res_stride();
    const int m = std::min(cap, stride);
    b200::orb::CamModel c{};
    if (cam) c = b200::orb::cam_model(*cam);
    b200_cv_keypoint_t* d_blob = nullptr;
    B200_CUDA(cudaMallocAsync((void**)&d_blob, sizeof(b200_cv_keypoint_t) * (size_t)std::max(m, 1), ex.stream));
    cudaError_t e = cudaSuccess;
    if (m > 0) {
        b200::orb::keyframe_blob_kernel<<<b200::ceil_div(m, 128), 128, 0, ex.stream>>>(c, cam ? 1 : 0, ex.res_kps() + (size_t)frame * stride,
                                                                                     ex.res_counts() + frame, m, d_blob);
        e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaMemcpyAsync(keypts_blob, d_blob, sizeof(b200_cv_keypoint_t) * (size_t)m, cudaMemcpyDeviceToHost, ex.stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(desc_blob, ex.res_descs() + (size_t)frame * stride * 32, (size_t)32 * m, cudaMemcpyDeviceToHost, ex.stream);
    }
    int count = 0;
    if (e == cudaSuccess) e = cudaMemcpyAsync(&count, ex.res_counts() + frame, sizeof(int), cudaMemcpyDeviceToHost, ex.stream);
    cudaFreeAsync(d_blob, ex.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ex.stream);
    if (e != cudaSuccess) return b200::cuda_fail(e, "b200_orb_export_keyframe_blobs", __FILE__, __LINE__);
    *n = count;
    if (count > cap) {
        b200::set_error("b200_orb_export_keyframe_blobs: frame %d has %d keypoints, cap is %d", frame, count, cap);
        return B200_ERR_CAPACITY;
    }
    return B200_OK;
}

int b200_rgbd_depths(b200_orb_t h, int n_frames, const b200_camera_intrinsics_t* cam, double focal_x_baseline, double depthmap_factor, int depth_type,
                     const void* depth_maps, int width, int height, size_t pitch, size_t frame_stride, int cap, b200_keypoint_t* undist_keypts,
                     double* bearings, float* depths, float* x_right, int32_t* n_keypoints) {
    B200_RANGE("b200:orb:rgbd_depths");
    if (!h || !cam || !n_keypoints || n_frames < 0 || cap < 0 || !b200::chain::camera_valid(*cam)) return B200_ERR_INVALID;
    Extractor& ex = h->ex;
    if (cam->model == 1) {
        b200::set_error("b200_rgbd_depths: an equirectangular camera has no RGB-D unprojection (data/common.cc:236-238 throws)");
        return B200_ERR_INVALID;
    }
    if (depth_type != B200_DEPTH_16UC1 && depth_type != B200_DEPTH_32FC1) {
        b200::set_error("b200_rgbd_depths: depth type %d is neither CV_16UC1 (%d) nor CV_32FC1 (%d)", depth_type, B200_DEPTH_16UC1, B200_DEPTH_32FC1);
        return B200_ERR_INVALID;
    }
    if (!(depthmap_factor > 0.0) || !std::isfinite(depthmap_factor)) {
        b200::set_error("b200_rgbd_depths: depthmap_factor must be positive and finite");
        return B200_ERR_INVALID;
    }
    if (n_frames == 0) return B200_OK;
    if (ex.width == 0 || n_frames > ex.last_batch) {
        b200::set_error("b200_rgbd_depths: %d frames requested, the last extract holds %d", n_frames, ex.last_batch);
        return B200_ERR_INVALID;
    }
    const size_t es = depth_type == B200_DEPTH_16UC1 ? 2 : 4, row = (size_t)width * es;
    if (width != ex.width || height != ex.height) {  // the reference only warns (is_valid_shape, system.cc:469-474) and then reads out of bounds
        b200::set_error("b200_rgbd_depths: depth map %dx%d, extracted frames %dx%d", width, height, ex.width, ex.height);
        return B200_ERR_INVALID;
    }
    if (!depth_maps || pitch < row || (n_frames > 1 && frame_stride < pitch * (size_t)height)
        || (cap > 0 && (!undist_keypts || !bearings || !depths || !x_right))) {
        b200::set_error("b200_rgbd_depths: invalid buffers");
        return B200_ERR_INVALID;
    }
    B200_CUDA(cudaSetDevice(ex.prm.device));
    cudaStream_t st = ex.stream;
    const size_t F = (size_t)n_frames, M = F * (size_t)cap, map_bytes = row * (size_t)height;
    b200::Layout L;
    const size_t o_map = L.take(map_bytes * F), o_kp = L.take<b200_keypoint_t>(M), o_b = L.take(24 * M), o_d = L.take(4 * M);
    const size_t o_xr = L.take(4 * M), o_n = L.take(4 * F);
    unsigned char* d = nullptr;
    B200_CUDA(cudaMallocAsync((void**)&d, L.end, st));
    const unsigned char* src = static_cast<const unsigned char*>(depth_maps);
    cudaError_t e = cudaSuccess;
    if (F == 1 || frame_stride == pitch * (size_t)height)
        e = cudaMemcpy2DAsync(d + o_map, row, src, pitch, row, (size_t)height * F, cudaMemcpyHostToDevice, st);
    else
        for (size_t f = 0; f < F && e == cudaSuccess; ++f)
            e = cudaMemcpy2DAsync(d + o_map + f * map_bytes, row, src + f * frame_stride, pitch, row, height, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d + o_n, ex.res_counts(), 4 * F, cudaMemcpyDeviceToDevice, st);
    if (e == cudaSuccess && cap > 0) {
        b200::orb::RgbdArgs a{};
        a.cam = b200::orb::cam_model(*cam);
        a.fxb = focal_x_baseline;
        a.scale = (float)(1.0 / depthmap_factor);
        a.is_16u = depth_type == B200_DEPTH_16UC1;
        a.copy = !a.is_16u && depthmap_factor == 1.0;
        a.w = width;
        a.h = height;
        a.pitch = row;
        a.fstride = map_bytes;
        a.kp_stride = ex.res_stride();
        a.cap = cap;
        b200::orb::rgbd_depths_kernel<<<dim3(b200::ceil_div(std::min(cap, a.kp_stride), 128), n_frames), 128, 0, st>>>(
            a, ex.res_kps(), (const int*)(d + o_n), d + o_map, (b200_keypoint_t*)(d + o_kp), (double*)(d + o_b), (float*)(d + o_d), (float*)(d + o_xr));
        e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaMemcpyAsync(undist_keypts, d + o_kp, sizeof(b200_keypoint_t) * M, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(bearings, d + o_b, 24 * M, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(depths, d + o_d, 4 * M, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(x_right, d + o_xr, 4 * M, cudaMemcpyDeviceToHost, st);
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(n_keypoints, d + o_n, 4 * F, cudaMemcpyDeviceToHost, st);
    cudaFreeAsync(d, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return b200::cuda_fail(e, "b200_rgbd_depths", __FILE__, __LINE__);
    for (int f = 0; f < n_frames; ++f)
        if (n_keypoints[f] > cap) {
            b200::set_error("b200_rgbd_depths: frame %d has %d keypoints, cap is %d", f, n_keypoints[f], cap);
            return B200_ERR_CAPACITY;
        }
    return B200_OK;
}

int b200_keyframe_blob_to_keypoints(const b200_cv_keypoint_t* keypts_blob, int n, b200_keypoint_t* keypts) {
    if (n < 0 || (n > 0 && (!keypts_blob || !keypts))) return B200_ERR_INVALID;
    for (int i = 0; i < n; ++i) {
        const b200_cv_keypoint_t& s = keypts_blob[i];
        b200_keypoint_t o;
        o.x = s.x; o.y = s.y; o.size = s.size; o.angle = s.angle; o.response = s.response; o.octave = s.octave;
        keypts[i] = o;
    }
    return B200_OK;
}

int b200_orb_raw_corner_counts(b200_orb_t h, int32_t* counts, int n) {
    if (!h || !counts || n < 0) return B200_ERR_INVALID;
    n = std::min(n, h->ex.last_batch);
    if (n == 0 || !h->ex.d_raw_corners) return B200_OK;
    B200_CUDA(cudaSetDevice(h->ex.prm.device));
    B200_CUDA(cudaMemcpyAsync(counts, h->ex.d_raw_corners, sizeof(int) * n, cudaMemcpyDeviceToHost, h->ex.stream));
    B200_CUDA(cudaStreamSynchronize(h->ex.stream));
    return B200_OK;
}

int b200_orb_stage_ms(b200_orb_t h, int stage, float* ms) {
    if (!h || !ms || stage < 0 || stage > 5) return B200_ERR_INVALID;
    *ms = h->ex.stage_ms[stage];
    return B200_OK;
}

}  // extern "C"

namespace b200 {
namespace chain {
int orb_results(b200_orb_t orb, const b200_keypoint_t** d_kps, const unsigned char** d_descs, const int** d_counts, int* stride, int* batch,
                cudaStream_t* stream, int* device) {
    if (!orb || orb->ex.width == 0 || orb->ex.last_batch <= 0) {
        set_error("b200_track_local_map: the extractor holds no results (call b200_orb_extract* first)");
        return B200_ERR_INVALID;
    }
    *d_kps = orb->ex.res_kps();
    *d_descs = orb->ex.res_descs();
    *d_counts = orb->ex.res_counts();
    *stride = orb->ex.res_stride();
    *batch = orb->ex.last_batch;
    *stream = orb->ex.stream;
    *device = orb->ex.prm.device;
    return B200_OK;
}
}  // namespace chain
}  // namespace b200
