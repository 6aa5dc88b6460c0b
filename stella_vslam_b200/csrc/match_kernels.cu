// match_kernels.cu -- 256-bit Hamming matchers on sm_90a.
//
// Reference path:
//   match::compute_descriptor_distance_32      src/stella_vslam/match/base.h:20-41
//   match::robust::brute_force_match           src/stella_vslam/match/robust.cc:232-328
//   util::angle::diff                          src/stella_vslam/util/angle.cc:7-16
//
// brute_force_match is sequential in the reference: keyframe keypoints idx_2 are visited in order and every accepted
// match removes its frame keypoint idx_1 from all later searches.  Restated here as
//   (1) a fully parallel pass that keeps, per idx_2, the K smallest (distance, idx_1) keys over the orientation-gated
//       frame keypoints (an int8 GEMM on the tensor cores, listing only distances that can still decide a match), and
//   (2) an in-order resolve (one warp per problem) that walks each list skipping taken idx_1; when a list cannot decide
//       the outcome exactly (too many of its entries were taken) the warp recomputes that row against the live set.
// Both steps are exact, so the match pairs equal the reference's bit for bit.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstddef>
#include <type_traits>
#include <new>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "essential_ransac.cuh"
#include "staging.cuh"
#include "track_chain.cuh"
#include "triangulate.cuh"

namespace b200 {
namespace match {

constexpr int kTopK = 8;            // candidates kept per keyframe keypoint
constexpr int kListRowAlign = 64;   // a problem's candidate lists are padded to a multiple of this many keyframe rows
constexpr unsigned kInfKey = 0xFFFFFFFFu;
constexpr unsigned kSentinelIdx = 0x3FFFFFu;  // index no keypoint can have (frames hold < 2^22 - 1 keypoints)
constexpr int kThrLow = 50;         // HAMMING_DIST_THR_LOW  (match/base.h:15)
constexpr int kMaxDist = 256;       // MAX_HAMMING_DIST      (match/base.h:17)

// key = distance << 22 | idx_1 : unsigned order == (distance, then first index) == the reference's strict '<' scan
__device__ __forceinline__ unsigned make_key(unsigned dist, unsigned idx) { return (dist << 22) | idx; }
__device__ __forceinline__ unsigned key_dist(unsigned key) { return key >> 22; }
__device__ __forceinline__ unsigned key_idx(unsigned key) { return key & 0x3FFFFFu; }

// util/angle.cc:7-16 compares and adds in double (float operands promoted).  With float operands these are the same decisions and the
// same values in float arithmetic: -180, 180, 360 and 30 are exact floats, promoting a float is exact (so the comparisons agree), and
// (float)((double)ret + 360.0) rounds an exactly representable double sum once -- which is what __fadd_rn(ret, 360.0f) does.  Float
// keeps the test off the fp64 pipe (it sits in the selection path of every matcher).
__device__ __forceinline__ float angle_diff(float a1, float a2) {
    float ret = __fsub_rn(a1, a2);
    if (ret <= -180.0f) ret = __fadd_rn(ret, 360.0f);
    if (ret > 180.0f) ret = __fsub_rn(ret, 360.0f);
    return ret;
}
__device__ __forceinline__ bool orientation_rejects(float a1, float a2) {  // robust.cc:279
    return fabsf(angle_diff(a1, a2)) > 30.0f;
}

__device__ __forceinline__ unsigned hamming256(const uint4& a0, const uint4& a1, const uint4& b0, const uint4& b1) {
    return __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) + __popc(a1.x ^ b1.x)
           + __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
}

// ---------------------------------------------------------------------------------------------------------------
// all-pairs distance matrix (diagnostics / landmark::compute_descriptor-style consumers)
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) hamming_matrix_kernel(const uint4* __restrict__ d1, int n1, const uint4* __restrict__ d2, int n2,
                                                             unsigned short* __restrict__ out) {
    __shared__ uint4 s2[64 * 2];
    const int j0 = blockIdx.x * 64, i = blockIdx.y * blockDim.x + threadIdx.x;
    for (int t = threadIdx.x; t < 128; t += blockDim.x) s2[t] = (j0 + t / 2 < n2) ? d2[(size_t)j0 * 2 + t] : make_uint4(0, 0, 0, 0);
    __syncthreads();
    if (i >= n1) return;
    const uint4 a0 = d1[(size_t)i * 2], a1 = d1[(size_t)i * 2 + 1];
    for (int j = 0; j < 64 && j0 + j < n2; ++j) out[(size_t)i * n2 + j0 + j] = (unsigned short)hamming256(a0, a1, s2[2 * j], s2[2 * j + 1]);
}

// ---------------------------------------------------------------------------------------------------------------
// the two sides of a batch of matching problems
// ---------------------------------------------------------------------------------------------------------------
struct Side {                       // one side of the problems: descriptors, strided angles, per-problem (offset, count)
    const uint4* desc;
    const unsigned char* angle;     // angle of keypoint i = *(const float*)(angle + i * angle_stride)
    long long angle_stride;
    const int* off;
    const int* cnt;
};
__device__ __forceinline__ float side_angle(const Side& s, int i) {
    return *reinterpret_cast<const float*>(s.angle + (long long)i * s.angle_stride);
}

// ---------------------------------------------------------------------------------------------------------------
// (1) top-K candidate lists on the Hopper tensor cores.  The Hamming distance of two 256-bit descriptors is a dot product in
//      disguise: with the bits mapped to +-1,  popcount(a ^ b) = (256 - <a, b>) / 2  -- exact in int32 -- so the all-pairs distance
//      matrix of a (frame, keyframe) pair is a 2000 x 2000 x 256 int8 GEMM.  One CTA owns 128 keyframe rows (the A operand, expanded
//      once into shared memory in the K-major no-swizzle core-matrix layout: 8 rows x 16 bytes per core matrix) and walks the frame's
//      keypoints in chunks of 128 (the B operand, expanded by the same threads into one of two buffers).  Each of the two warpgroups
//      issues wgmma.mma_async.m64n128k32.s32.s8.s8 (8 per chunk) for its 64 rows with the accumulators in registers; while the tensor
//      core works on chunk c the threads expand chunk c+1 into the other buffer, then every thread scans its accumulator fragment (two
//      rows x 32 columns) and keeps, per row, the kTopK smallest (distance, index) keys that pass the orientation gate, among the
//      distances up to a cap that cannot change a decision.  The four lanes of a quad hold the same two rows; their lists
//      are merged at the end.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kTcRows = 128;        // keyframe rows per CTA (two m64 tiles); two CTAs share an SM: one stages / waits while the other selects
constexpr int kTcChunk = 128;       // frame keypoints per B chunk (= N of the MMA)
constexpr int kTcThreads = 256;     // two warpgroups, one per 64-row half of the A tile
constexpr int kTcTileBytes = 128 * 256;  // one 128-row operand tile of +-1 bytes
struct TcSmem {
    unsigned char a[kTcTileBytes];
    unsigned char b[2][kTcTileBytes];
    uint2 lut[256];                 // descriptor byte -> 8 bytes of +-1
    float ang[2][kTcChunk];
};
__device__ __forceinline__ unsigned long long gmma_desc_k_major(unsigned smem_addr, unsigned lbo_bytes, unsigned sbo_bytes) {
    // wgmma matrix descriptor: start address [0,14), leading byte offset [16,30), stride byte offset [32,46) (all >> 4), base offset 0,
    // layout type 0 (no swizzle) at [62,64).  K-major canonical layout ((8,m),2):((1,SBO),LBO) in 16-byte units.
    return (unsigned long long)((smem_addr >> 4) & 0x3FFFu) | ((unsigned long long)((lbo_bytes >> 4) & 0x3FFFu) << 16)
           | ((unsigned long long)((sbo_bytes >> 4) & 0x3FFFu) << 32);
}
// D (64 x 128, s32) [+]= A (64 x 32, s8, K-major) * B (128 x 32, s8, K-major)^T; thread t of the warpgroup holds rows
// 16 (t / 32) + (t % 32) / 4 (+ 8) and columns 8 i + 2 (t % 4) (+ 1): d[4 i + {0, 1}] row r, d[4 i + {2, 3}] row r + 8
__device__ __forceinline__ void wgmma_s8_m64n128k32(unsigned (&d)[64], unsigned long long da, unsigned long long db, unsigned accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, "
        "%18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, "
        "%45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p;\n\t}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]),
          "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]),
          "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]),
          "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]),
          "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]),
          "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]),
          "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
        : "l"(da), "l"(db), "r"(accumulate)
        : "memory");
}
// keeps the compiler from moving reads or writes of the accumulators across the wgmma fence / wait instructions
__device__ __forceinline__ void wgmma_fence_operands(unsigned (&d)[64]) {
#pragma unroll
    for (int i = 0; i < 64; ++i) asm volatile("" : "+r"(d[i])::"memory");
}
// +-1 expansion of one 16-byte half descriptor (8 K-chunks of 16 bytes) into the operand tile: row r of a 128-row tile, chunks c0..c0+7
__device__ __forceinline__ void tc_expand_half(unsigned char* tile, const uint2* lut, int r, int c0, uint4 bits) {
    unsigned char* dst = tile + (r >> 3) * 128 + (r & 7) * 16;
    const unsigned w[4] = {bits.x, bits.y, bits.z, bits.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) {  // chunk c0 + i <- descriptor bytes 2i, 2i+1 of this half
        const unsigned hw = (w[i >> 1] >> (16 * (i & 1))) & 0xFFFFu;
        const uint2 lo = lut[hw & 0xFFu], hi = lut[hw >> 8];
        *reinterpret_cast<uint4*>(dst + (c0 + i) * 2048) = make_uint4(lo.x, lo.y, hi.x, hi.y);
    }
}
__device__ __forceinline__ void tc_zero_half(unsigned char* tile, int r, int c0) {
    unsigned char* dst = tile + (r >> 3) * 128 + (r & 7) * 16;
#pragma unroll
    for (int i = 0; i < 8; ++i) *reinterpret_cast<uint4*>(dst + (c0 + i) * 2048) = make_uint4(0, 0, 0, 0);
}
__device__ __forceinline__ void insert_key(unsigned (&top)[kTopK], unsigned key) {
    top[kTopK - 1] = key;
#pragma unroll
    for (int k = kTopK - 1; k > 0; --k) {
        if (top[k] < top[k - 1]) {
            const unsigned t = top[k];
            top[k] = top[k - 1];
            top[k - 1] = t;
        }
    }
}

__global__ void __launch_bounds__(kTcThreads, 2) topk_tc_kernel(Side S1, Side S2, const unsigned char* __restrict__ valid2, int check_orientation,
                                                                unsigned* __restrict__ lists, int list_rows, unsigned cap) {
    extern __shared__ __align__(1024) unsigned char tc_smem_raw[];
    TcSmem& sm = *reinterpret_cast<TcSmem*>(tc_smem_raw);
    const uint4* __restrict__ desc1 = S1.desc;
    const uint4* __restrict__ desc2 = S2.desc;
    const int p = blockIdx.y;
    const int b1 = S1.off[p], n1 = S1.cnt[p];
    const int b2 = S2.off[p], n2 = S2.cnt[p];
    const int row0 = blockIdx.x * kTcRows;
    if (row0 >= n2) return;
    const int tid = threadIdx.x, lane = tid & 31;
    for (int e = tid; e < 256; e += kTcThreads) {  // bit i of the byte -> byte i: +1 (0x01) if set, -1 (0xFF) if clear
        unsigned lo = 0, hi = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            lo |= (((e >> i) & 1) ? 0x01u : 0xFFu) << (8 * i);
            hi |= (((e >> (4 + i)) & 1) ? 0x01u : 0xFFu) << (8 * i);
        }
        sm.lut[e] = make_uint2(lo, hi);
    }
    __syncthreads();
    // staging: thread = (operand row, descriptor half); each thread expands ONE 16-byte half of a row (8 of the 16 K-chunks)
    const int rtid = tid & 127, half = tid >> 7;
    if (row0 + rtid < n2) tc_expand_half(sm.a, sm.lut, rtid, 8 * half, desc2[(size_t)(b2 + row0 + rtid) * 2 + half]);
    else tc_zero_half(sm.a, rtid, 8 * half);  // rows past the keyframe: zeros (their lists are never written)
    // selection: warpgroup wg = half owns A rows 64 wg .. 64 wg + 63; this thread's two rows are r_lo and r_lo + 8
    const int r_lo = 64 * half + 16 * ((tid >> 5) & 3) + (lane >> 2);
    bool active[2];
    float qa[2];
    unsigned thr[2], top[2][kTopK];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int row = row0 + r_lo + 8 * h;
        active[h] = row < n2 && (!valid2 || valid2[b2 + row]);
        qa[h] = active[h] ? side_angle(S2, b2 + row) : 0.f;
        // Distance cap.  robust.cc:297-308 accepts a match only if best <= 50 and lowe * second >= best, so a second-best distance
        // matters only while lowe * second < 50: a candidate farther than cap = ceil(50 / lowe) can change no decision and is not listed
        // (random descriptor pairs are ~128 +- 8 apart, so this removes nearly every insertion).  Rows without a landmark list nothing.
        thr[h] = active[h] ? make_key(cap + 1u, 0u) : 0u;
#pragma unroll
        for (int k = 0; k < kTopK; ++k) top[h][k] = kInfKey;
    }
    const unsigned a_addr = (unsigned)__cvta_generic_to_shared(sm.a) + (unsigned)(half * 8 * 128);
    const unsigned b_addr[2] = {(unsigned)__cvta_generic_to_shared(sm.b[0]), (unsigned)__cvta_generic_to_shared(sm.b[1])};
    const int n_chunks = (n1 + kTcChunk - 1) / kTcChunk;
    // B operand of a chunk: 128 frame keypoints, thread = (row, half).  The descriptor bits (and angle) of the NEXT chunk are fetched one
    // chunk ahead, so the L2 latency hides behind the tensor core and the selection pass.
    uint4 nb = make_uint4(0, 0, 0, 0);
    float nang = 0.f;
    auto fetch = [&](int j) {
        if (j < n1) {
            nb = desc1[(size_t)(b1 + j) * 2 + half];
            if (half == 0) nang = side_angle(S1, b1 + j);
        }
    };
    auto stage = [&](int c) {
        const int j = c * kTcChunk + rtid;
        if (j < n1) {
            tc_expand_half(sm.b[c & 1], sm.lut, rtid, 8 * half, nb);
            if (half == 0) sm.ang[c & 1][rtid] = nang;
        } else {
            tc_zero_half(sm.b[c & 1], rtid, 8 * half);
        }
        fetch(j + kTcChunk);
    };
    fetch(rtid);
    if (n_chunks > 0) stage(0);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> visible to the tensor core's async proxy
    __syncthreads();
    unsigned acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0u;
    for (int c = 0; c < n_chunks; ++c) {
        const int buf = c & 1, c0 = c * kTcChunk;
        wgmma_fence_operands(acc);
        asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
        for (int ks = 0; ks < 8; ++ks)  // K = 32 bytes per instruction = chunks 2 ks, 2 ks + 1 (2048 bytes apart)
            wgmma_s8_m64n128k32(acc, gmma_desc_k_major(a_addr + ks * 4096, 2048, 128), gmma_desc_k_major(b_addr[buf] + ks * 4096, 2048, 128),
                                ks > 0 ? 1u : 0u);
        asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
        if (c + 1 < n_chunks) {  // chunk c + 1 into the other buffer while the tensor core works on chunk c
            stage(c + 1);
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        }
        asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
        wgmma_fence_operands(acc);
        // key = distance << 22 | index with distance = (256 - dot) / 2:  (256 - dot) << 21 has bit 21 clear (the dot product of two
        // +-1 vectors of even length is even), so the key is one multiply-add.  The four keys of a column pair (two per row) are tested
        // against the rows' thresholds with one warp vote; only a group that holds a candidate for some row of the warp inserts.  The
        // thresholds start at the distance cap, so candidates are rare: a warp's 16 rows see a few dozen in all.
        const unsigned kbase = (256u << 21) + (unsigned)c0;
        auto scan = [&](auto full_chunk) {
#pragma unroll
            for (int i = 0; i < kTcChunk / 8; ++i) {
                const int col = 8 * i + 2 * (lane & 3);
                unsigned key[2][2];
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int u = 0; u < 2; ++u) {
                        key[h][u] = (unsigned)((int)acc[4 * i + 2 * h + u] * -(1 << 21)) + (kbase + (unsigned)(col + u));
                        if (!decltype(full_chunk)::value && c0 + col + u >= n1) key[h][u] = kInfKey;  // zero padding of the last chunk
                    }
                const bool hit = min(key[0][0], key[0][1]) < thr[0] || min(key[1][0], key[1][1]) < thr[1];
                if (__any_sync(0xFFFFFFFFu, hit)) {
#pragma unroll
                    for (int h = 0; h < 2; ++h)
#pragma unroll
                        for (int u = 0; u < 2; ++u) {
                            if (key[h][u] < thr[h]) {
                                if (check_orientation && orientation_rejects(sm.ang[buf][col + u], qa[h])) continue;
                                insert_key(top[h], key[h][u]);
                                thr[h] = min(thr[h], top[h][kTopK - 1]);
                            }
                        }
                }
            }
        };
        if (c0 + kTcChunk <= n1) scan(std::true_type{});
        else scan(std::false_type{});
        __syncthreads();  // chunk c + 1 is staged; nobody reads chunk c's buffer or angles any more
    }
    // merge the four quad lists of every row: each thread parks its (sorted) lists in the B staging area (free: every warpgroup has
    // waited for its last MMA before the loop's closing barrier), one thread per row merges
    unsigned* park = reinterpret_cast<unsigned*>(sm.b[0]);
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int k = 0; k < kTopK; ++k) park[((r_lo + 8 * h) * 4 + (lane & 3)) * kTopK + k] = top[h][k];
    __syncthreads();
    if (tid < kTcRows) {
        unsigned t[kTopK];
#pragma unroll
        for (int k = 0; k < kTopK; ++k) t[k] = park[tid * 4 * kTopK + k];
        for (int q = 1; q < 4; ++q) {
#pragma unroll
            for (int k2 = 0; k2 < kTopK; ++k2) {
                const unsigned key = park[(tid * 4 + q) * kTopK + k2];
                if (key < t[kTopK - 1]) insert_key(t, key);
            }
        }
        // lists shorter than 8: the slots name no candidate but state the bound "everything else is farther than the cap"
#pragma unroll
        for (int k = 0; k < kTopK; ++k)
            if (t[k] == kInfKey && cap < (unsigned)kMaxDist) t[k] = make_key(cap + 1u, kSentinelIdx);
        if (row0 + tid < n2) {
            unsigned* o = lists + ((size_t)p * list_rows + row0 + tid) * kTopK;
#pragma unroll
            for (int k = 0; k < kTopK; ++k) o[k] = t[k];
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// (2) in-order resolve + compaction.  One warp per problem.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned warp_min(unsigned v) {
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) v = min(v, __shfl_xor_sync(0xFFFFFFFFu, v, s));
    return v;
}

// exact best/second over the live (not taken, orientation-gated) frame keypoints: the reference's inner loop, one warp.
// desc1/angle1 point either to the problem's frame side in global memory (angle stride in bytes) or to its staged copy in
// shared memory.
__device__ void exact_row(const uint4* desc1, const unsigned char* angle1, long long angle_stride, int n1, const volatile unsigned* taken,
                          uint4 q0, uint4 q1, float qa, int check_orientation, int lane, unsigned* best_key, unsigned* second_dist) {
    unsigned k1 = kInfKey, k2 = kInfKey;  // two smallest keys seen by this lane
    for (int i0 = lane; i0 < n1; i0 += 128) {
        uint4 a0[4], a1[4];
        float ang[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {  // four independent loads in flight per lane
            const int i = min(i0 + 32 * u, n1 - 1);
            a0[u] = desc1[(size_t)i * 2];
            a1[u] = desc1[(size_t)i * 2 + 1];
            ang[u] = *reinterpret_cast<const float*>(angle1 + (long long)i * angle_stride);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int i = i0 + 32 * u;
            if (i >= n1) continue;
            if ((taken[i >> 5] >> (i & 31)) & 1u) continue;
            if (check_orientation && orientation_rejects(ang[u], qa)) continue;
            const unsigned key = make_key(hamming256(q0, q1, a0[u], a1[u]), (unsigned)i);
            if (key < k1) {
                k2 = k1;
                k1 = key;
            } else if (key < k2) {
                k2 = key;
            }
        }
    }
    const unsigned b = warp_min(k1);
    const unsigned mine = (k1 == b) ? k2 : k1;  // keys are unique (they embed idx_1), so exactly one lane owns b
    const unsigned s = warp_min(mine);
    *best_key = b;
    *second_dist = (s == kInfKey) ? (unsigned)kMaxDist : key_dist(s);
}

// Decision of one keyframe keypoint from its sorted candidate list against the current `taken` set.
//   returns 0: decided, no match; 1: decided, match with key *best; 2: undecidable from the list (exact row scan needed)
__device__ __forceinline__ int decide_row(const unsigned (&keys)[kTopK], bool full, unsigned tail_dist, const volatile unsigned* taken, float lowe_ratio,
                                          unsigned* best) {
    unsigned best_key = kInfKey, second_dist = kMaxDist;
    int n_live = 0;
#pragma unroll
    for (int k = 0; k < kTopK; ++k) {
        const unsigned key = keys[k];
        if (key == kInfKey) continue;
        const unsigned i1 = key_idx(key);
        if ((taken[i1 >> 5] >> (i1 & 31)) & 1u) continue;
        if (n_live == 0) best_key = key;
        else if (n_live == 1) second_dist = key_dist(key);
        ++n_live;
    }
    // full: unlisted candidates exist; every unlisted distance is >= tail_dist
    if (full && n_live < 2) {
        if (n_live == 1) {
            // best is exact; the true second distance lies in [tail_dist, 256]
            const unsigned bd = key_dist(best_key);
            if (bd > (unsigned)kThrLow) return 0;
            if (__fmul_rn(lowe_ratio, (float)tail_dist) < (float)bd) return 2;
            second_dist = tail_dist;  // passes the ratio test even with the smallest possible second distance
        } else {
            // every listed candidate is taken: the best live distance is >= tail_dist
            return (tail_dist > (unsigned)kThrLow) ? 0 : 2;
        }
    }
    if (best_key == kInfKey) return 0;
    const unsigned bd = key_dist(best_key);
    // robust.cc:297-308: threshold, then Lowe ratio in float
    if (bd > (unsigned)kThrLow || __fmul_rn(lowe_ratio, (float)second_dist) < (float)bd) return 0;
    *best = best_key;
    return 1;
}

// One warp per problem.  Rows (keyframe keypoints) are visited in batches of 32, one per lane.  Every lane decides its row
// against the taken set as of the last commit; a lane's decision is final iff no earlier, not yet committed lane accepts a
// frame keypoint that appears in its candidate list -- so the longest conflict-free prefix of the batch is committed at
// once and the rest re-decided.  The result is identical to the reference's strictly sequential loop.
__global__ void __launch_bounds__(32) resolve_kernel(Side S1, Side S2, const unsigned char* __restrict__ valid2,
                                                     const unsigned* __restrict__ lists, float lowe_ratio, int check_orientation,
                                                     int* __restrict__ matched, unsigned* __restrict__ taken_g, int taken_words,
                                                     int list_rows, int matched_stride, int pairs_stride,
                                                     int* __restrict__ pairs_out, int* __restrict__ n_pairs, int use_smem) {
    const uint4* __restrict__ desc1 = S1.desc;
    const uint4* __restrict__ desc2 = S2.desc;
    extern __shared__ __align__(16) unsigned resolve_smem[];  // [desc1 copy 32 B x n][angles][taken bitmap][idx_1 -> idx_2 table][claim table], as far as they fit
    const int p = blockIdx.x, lane = threadIdx.x;
    const int b1 = S1.off[p], n1 = S1.cnt[p];
    const int b2 = S2.off[p], n2 = S2.cnt[p];
    // the sequential state lives in shared memory (30-cycle instead of L2 latency on the critical path); very large frames fall
    // back to the global scratch
    // use_smem: 0 = everything in global scratch, 1 = taken + table in shared memory, 2 = additionally the frame descriptors and
    // angles (the exact fallback then scans shared memory instead of L2)
    const int stage_words = (use_smem == 2) ? 9 * matched_stride : 0;  // 8 words of descriptor + 1 angle per keypoint
    unsigned* taken = use_smem ? resolve_smem + stage_words : taken_g + (size_t)p * taken_words;
    int* m21 = use_smem ? reinterpret_cast<int*>(resolve_smem + stage_words + taken_words) : matched + (size_t)p * matched_stride;
    int* claim = use_smem ? reinterpret_cast<int*>(resolve_smem + stage_words + taken_words + matched_stride) : nullptr;
    int* pairs = pairs_out + 2 * (size_t)p * pairs_stride;
    lists += (size_t)p * list_rows * kTopK;
    for (int i = lane; i < (n1 + 31) / 32; i += 32) taken[i] = 0u;
    for (int i = lane; i < n1; i += 32) m21[i] = -1;
    if (claim)
        for (int i = lane; i < n1; i += 32) claim[i] = 255;
    __syncwarp();
    const uint4* d1 = desc1 + (size_t)b1 * 2;
    const unsigned char* a1p = S1.angle + (long long)b1 * S1.angle_stride;
    long long a1s = S1.angle_stride;
    if (use_smem == 2) {
        uint4* sd = reinterpret_cast<uint4*>(resolve_smem);
        float* sa = reinterpret_cast<float*>(resolve_smem + 8 * matched_stride);
        for (int i = lane; i < 2 * n1; i += 32) sd[i] = d1[i];
        for (int i = lane; i < n1; i += 32) sa[i] = side_angle(S1, b1 + i);
        d1 = sd;
        a1p = reinterpret_cast<const unsigned char*>(sa);
        a1s = sizeof(float);
        __syncwarp();
    }
    for (int base = 0; base < n2; base += 32) {
        const int r = base + lane;
        const bool has_row = r < n2 && (!valid2 || valid2[b2 + r]);  // robust.cc:255-262
        unsigned keys[kTopK];
        {
            const uint4* lp = reinterpret_cast<const uint4*>(lists + (size_t)min(r, n2 - 1) * kTopK);
            const uint4 k0 = lp[0], k1 = lp[1];
            keys[0] = k0.x; keys[1] = k0.y; keys[2] = k0.z; keys[3] = k0.w;
            keys[4] = k1.x; keys[5] = k1.y; keys[6] = k1.z; keys[7] = k1.w;
        }
        // A list is "full" when candidates exist that it does not name: its last entry then bounds their distance from below.  The
        // tensor-core lister only names candidates up to a distance cap and pads with sentinel keys (cap + 1, impossible index).
        const bool list_full = keys[kTopK - 1] != kInfKey;
        const unsigned tail_dist = key_dist(keys[kTopK - 1]);
#pragma unroll
        for (int k = 0; k < kTopK; ++k)
            if (key_idx(keys[k]) == kSentinelIdx) keys[k] = kInfKey;
        unsigned pending = __ballot_sync(0xFFFFFFFFu, has_row);
        while (pending) {
            const bool mine = (pending >> lane) & 1u;
            unsigned best = kInfKey;
            const int st = mine ? decide_row(keys, list_full, tail_dist, taken, lowe_ratio, &best) : 0;
            const unsigned accept_mask = __ballot_sync(0xFFFFFFFFu, mine && st == 1);
            const unsigned exact_mask = __ballot_sync(0xFFFFFFFFu, mine && st == 2);
            // conflicts with earlier accepting lanes of this round
            bool conflict = false;
            const unsigned my_best_idx = key_idx(best);
            if (claim) {
                // claim[i] = lowest lane that accepts frame keypoint i this round; a lane conflicts when a lower lane claims any
                // keypoint of its list (8 shared-memory probes instead of one shuffle round per accepting lane)
                if (mine && st == 1) atomicMin(&claim[my_best_idx], lane);
                __syncwarp();
                if (mine) {
#pragma unroll
                    for (int k = 0; k < kTopK; ++k) conflict |= (keys[k] != kInfKey && claim[key_idx(keys[k])] < lane);
                }
                __syncwarp();
                if (mine && st == 1) claim[my_best_idx] = 255;
            } else {
                for (unsigned m = accept_mask; m; m &= m - 1) {
                    const int jl = __ffs(m) - 1;
                    const unsigned bj = __shfl_sync(0xFFFFFFFFu, my_best_idx, jl);
                    if (mine && lane > jl) {
#pragma unroll
                        for (int k = 0; k < kTopK; ++k) conflict |= (keys[k] != kInfKey && key_idx(keys[k]) == bj);
                    }
                }
            }
            const unsigned unsafe = __ballot_sync(0xFFFFFFFFu, mine && (conflict || st == 2));
            const int first_unsafe = unsafe ? __ffs(unsafe) - 1 : 32;
            const unsigned commit = pending & ((first_unsafe >= 32) ? 0xFFFFFFFFu : ((1u << first_unsafe) - 1u));
            if (((commit >> lane) & 1u) && st == 1) {
                const unsigned i1 = key_idx(best);
                atomicOr(&taken[i1 >> 5], 1u << (i1 & 31));  // distinct lanes may share a word
                m21[i1] = r;
            }
            pending &= ~commit;
            __syncwarp();
            if (first_unsafe < 32 && ((exact_mask >> first_unsafe) & 1u) && !(((unsafe & ((1u << first_unsafe) - 1u)) != 0u))) {
                // the first not-yet-committed row cannot be decided from its list: warp-cooperative exact scan (the reference's inner loop)
                const int rr = base + first_unsafe;
                unsigned bk, sd;
                exact_row(d1, a1p, a1s, n1, taken, desc2[(size_t)(b2 + rr) * 2], desc2[(size_t)(b2 + rr) * 2 + 1], side_angle(S2, b2 + rr),
                          check_orientation, lane, &bk, &sd);
                if (bk != kInfKey) {
                    const unsigned bd = key_dist(bk);
                    if (!(bd > (unsigned)kThrLow) && !(__fmul_rn(lowe_ratio, (float)sd) < (float)bd)) {
                        const unsigned i1 = key_idx(bk);
                        if (lane == 0) {
                            taken[i1 >> 5] |= 1u << (i1 & 31);
                            m21[i1] = rr;
                        }
                    }
                }
                pending &= ~(1u << first_unsafe);
                __syncwarp();
            }
        }
    }
    __syncwarp();
    // robust.cc:317-325: pairs sorted by idx_1
    int total = 0;
    for (int base = 0; base < n1; base += 32) {
        const int i = base + lane;
        const int v = (i < n1) ? m21[i] : -1;
        const unsigned bal = __ballot_sync(0xFFFFFFFFu, v >= 0);
        if (v >= 0) {
            const int pos = total + __popc(bal & ((1u << lane) - 1u));
            pairs[2 * (size_t)pos] = i;
            pairs[2 * (size_t)pos + 1] = v;
        }
        total += __popc(bal);
    }
    if (lane == 0) n_pairs[p] = total;
}

// ---------------------------------------------------------------------------------------------------------------
// Grid-guided projection matchers
//   match::projection::match_frame_and_landmarks      src/stella_vslam/match/projection.cc:13-93    (mode 0)
//   match::projection::match_current_and_last_frames  src/stella_vslam/match/projection.cc:95-207   (mode 1)
//   data::assign_keypoints_to_grid / get_keypoints_in_cell   src/stella_vslam/data/common.cc:83-190, data/common.h:60-68
// G1 builds the keypoint grid (cell-x major, indices ascending inside a cell = the reference's iteration order), G2 lets one
// thread per landmark enumerate its search window in that order and record (distance, octave, index) for every candidate
// that passes the static gates, G3 replays the reference's sequential loop (a match removes the keypoint from all later
// searches) with the same prefix-commit scheme as the brute-force resolve.
// ---------------------------------------------------------------------------------------------------------------
struct GuidedDev {
    int n_train, n_queries, grid_cols, grid_rows, cap;
    float min_x, max_x, min_y, max_y;
    const float *t_x, *t_y, *t_angle, *t_x_right;
    const unsigned char* t_octave;
    const uint4* t_desc;
    const uint4* q_desc;
    const float *q_x, *q_y, *q_margin, *q_x_right, *q_angle;
    const signed char *q_min_level, *q_max_level;
    const unsigned char* q_valid;
    const double* q_reproj;           // mode 3
    const float* inv_level_sigma_sq;  // mode 3, 256 entries
    int do_reproj;
    // scratch + outputs of this problem
    int *cell_start, *cell_items, *cell_cursor, *owner;
    uint2* lists;
    int* list_len;
    unsigned char* occupied;
    int* match_out;
    int* n_matches;
};

__device__ __forceinline__ int cell_index(const GuidedDev& g, float x, float y, double inv_w, double inv_h) {
    const int cx = __double2int_rd((double)__fsub_rn(x, g.min_x) * inv_w), cy = __double2int_rd((double)__fsub_rn(y, g.min_y) * inv_h);
    return (0 <= cx && cx < g.grid_cols && 0 <= cy && cy < g.grid_rows) ? cx * g.grid_rows + cy : -1;
}

// G1: one CTA.  cell_start[c .. c+1) delimits the ascending keypoint indices of cell c (cell = cx * rows + cy).
__global__ void __launch_bounds__(1024) guided_grid_kernel(const GuidedDev* __restrict__ gs) {
    const GuidedDev g = gs[blockIdx.x];
    int *cell_start = g.cell_start, *cell_items = g.cell_items, *cell_cursor = g.cell_cursor;
    const int n_cells = g.grid_cols * g.grid_rows;
    const double inv_w = (double)g.grid_cols / (double)__fsub_rn(g.max_x, g.min_x), inv_h = (double)g.grid_rows / (double)__fsub_rn(g.max_y, g.min_y);
    for (int c = threadIdx.x; c <= n_cells; c += blockDim.x) cell_start[c] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < g.n_train; i += blockDim.x) {
        const int c = cell_index(g, g.t_x[i], g.t_y[i], inv_w, inv_h);
        if (c >= 0) atomicAdd(&cell_start[c + 1], 1);
    }
    __syncthreads();
    {  // running sum over the n_cells + 1 counters (block-wide: a contiguous chunk per thread, shuffle scan of the chunk sums).  A single
       // thread walking the 3 073 cells of the 64 x 48 grid was most of this kernel's time.
        __shared__ int warp_tot[32];
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        const int per = (n_cells + 1 + (int)blockDim.x - 1) / (int)blockDim.x;
        const int beg = min((int)threadIdx.x * per, n_cells + 1), end = min(beg + per, n_cells + 1);
        int sum = 0;
        for (int c = beg; c < end; ++c) sum += cell_start[c];
        int incl = sum;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const int v = __shfl_up_sync(0xFFFFFFFFu, incl, off);
            if (lane >= off) incl += v;
        }
        if (lane == 31) warp_tot[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            int w = lane < (int)(blockDim.x >> 5) ? warp_tot[lane] : 0;
#pragma unroll
            for (int off = 1; off < 32; off <<= 1) {
                const int v = __shfl_up_sync(0xFFFFFFFFu, w, off);
                if (lane >= off) w += v;
            }
            warp_tot[lane] = w;
        }
        __syncthreads();
        int run = incl - sum + (warp > 0 ? warp_tot[warp - 1] : 0);
        for (int c = beg; c < end; ++c) {
            run += cell_start[c];
            cell_start[c] = run;
        }
    }
    __syncthreads();
    for (int c = threadIdx.x; c < n_cells; c += blockDim.x) cell_cursor[c] = cell_start[c];
    __syncthreads();
    for (int i = threadIdx.x; i < g.n_train; i += blockDim.x) {
        const int c = cell_index(g, g.t_x[i], g.t_y[i], inv_w, inv_h);
        if (c >= 0) cell_items[atomicAdd(&cell_cursor[c], 1)] = i;
    }
    __syncthreads();
    for (int c = threadIdx.x; c < n_cells; c += blockDim.x) {  // restore ascending index order inside each (short) cell list
        const int a = cell_start[c], b = cell_start[c + 1];
        for (int i = a + 1; i < b; ++i) {
            const int v = cell_items[i];
            int j = i - 1;
            while (j >= a && cell_items[j] > v) {
                cell_items[j + 1] = cell_items[j];
                --j;
            }
            cell_items[j + 1] = v;
        }
    }
}

// G2: one thread per landmark: enumerate the window, apply the static gates, record candidates in iteration order.
// entry = distance << 8 | octave, idx
__global__ void __launch_bounds__(128) guided_candidates_kernel(const GuidedDev* __restrict__ gs, int mode, int check_orientation,
                                                                int* __restrict__ overflow) {
    const GuidedDev g = gs[blockIdx.y];
    const int *cell_start = g.cell_start, *cell_items = g.cell_items;
    uint2* lists = g.lists;
    int* list_len = g.list_len;
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= g.n_queries) return;
    int len = 0;
    if (!g.q_valid || (g.q_valid[q] & 1)) {
        const double inv_w = (double)g.grid_cols / (double)__fsub_rn(g.max_x, g.min_x), inv_h = (double)g.grid_rows / (double)__fsub_rn(g.max_y, g.min_y);
        const float ref_x = g.q_x[q], ref_y = g.q_y[q], margin = g.q_margin[q];
        const int min_level = g.q_min_level[q], max_level = g.q_max_level[q];
        // data/common.cc:137-155
        const int min_cx = max(0, __double2int_rd((double)__fsub_rn(__fsub_rn(ref_x, g.min_x), margin) * inv_w));
        const int max_cx = min(g.grid_cols - 1, __double2int_ru((double)__fadd_rn(__fsub_rn(ref_x, g.min_x), margin) * inv_w));
        const int min_cy = max(0, __double2int_rd((double)__fsub_rn(__fsub_rn(ref_y, g.min_y), margin) * inv_h));
        const int max_cy = min(g.grid_rows - 1, __double2int_ru((double)__fadd_rn(__fsub_rn(ref_y, g.min_y), margin) * inv_h));
        if (min_cx < g.grid_cols && max_cx >= 0 && min_cy < g.grid_rows && max_cy >= 0) {
            const uint4 q0 = g.q_desc[(size_t)q * 2], q1 = g.q_desc[(size_t)q * 2 + 1];
            uint2* out = lists + (size_t)q * g.cap;
            for (int cx = min_cx; cx <= max_cx; ++cx)
                for (int cy = min_cy; cy <= max_cy; ++cy) {
                    const int c = cx * g.grid_rows + cy;
                    for (int k = cell_start[c]; k < cell_start[c + 1]; ++k) {
                        const int idx = cell_items[k];
                        const int oct = g.t_octave[idx];
                        if (0 <= min_level && oct < min_level) continue;
                        if (0 <= max_level && max_level < oct) continue;
                        const float dx = __fsub_rn(g.t_x[idx], ref_x), dy = __fsub_rn(g.t_y[idx], ref_y);
                        if (!(fabsf(dx) < margin && fabsf(dy) < margin)) continue;
                        if (mode <= 1 && g.t_x_right) {  // stereo gate (projection.cc:56-61, 168-173)
                            const float xr = g.t_x_right[idx];
                            if (0.f < xr && margin < fabsf(__fsub_rn(g.q_x_right[q], xr))) continue;
                        }
                        if ((mode == 1 || mode == 4) && check_orientation && orientation_rejects(g.q_angle[q], g.t_angle[idx])) continue;
                        if (mode == 3 && g.do_reproj) {  // chi-square reprojection gate (fuse.cc:93-120), evaluated like the reference: double
                            const double e_x = __dsub_rn(g.q_reproj[2 * q], (double)g.t_x[idx]), e_y = __dsub_rn(g.q_reproj[2 * q + 1], (double)g.t_y[idx]);
                            double err_sq = __dadd_rn(__dmul_rn(e_x, e_x), __dmul_rn(e_y, e_y));
                            float chi_sq = 5.99146f;
                            if (g.t_x_right && g.t_x_right[idx] >= 0.f) {
                                const float e_xr = __fsub_rn(g.q_x_right[q], g.t_x_right[idx]);
                                err_sq = __dadd_rn(err_sq, (double)__fmul_rn(e_xr, e_xr));
                                chi_sq = 7.81473f;
                            }
                            if ((double)chi_sq < __dmul_rn(err_sq, (double)g.inv_level_sigma_sq[oct])) continue;
                        }
                        const unsigned d = hamming256(q0, q1, g.t_desc[(size_t)idx * 2], g.t_desc[(size_t)idx * 2 + 1]);
                        if (len < g.cap) out[len] = make_uint2((d << 8) | (unsigned)oct, (unsigned)idx);
                        ++len;
                    }
                }
        }
    }
    if (len > g.cap) {
        atomicMax(overflow, len);
        len = g.cap;
    }
    list_len[q] = len;
}

// the reference's best / second update in iteration order over the keypoints whose state admits the candidate
// (state: 0 = occupied, 0xFFFF = free; mode 4: Hamming distance of the match the keypoint currently holds, area.cc:49-51).
// Returns the accepted index or -1; *best_out = its distance.
__device__ __forceinline__ int guided_decide(const uint2* __restrict__ list, int len, const volatile unsigned short* state, int mode, unsigned thr,
                                             float lowe_ratio, unsigned* best_out) {
    // mode 5: bow_tree::match_frame_and_keyframe / match_keyframes; mode 6: match_for_triangulation, whose running best starts at
    // the threshold and which skips every candidate above it (robust.cc:57-59, 83-85)
    unsigned best = mode == 6 ? thr : (unsigned)kMaxDist, second = kMaxDist;
    int best_level = -1, second_level = -1, best_idx = -1;
    const bool track_second = mode == 0 || mode >= 4;
    for (int k = 0; k < len; ++k) {
        const uint2 e = list[k];
        const unsigned idx = e.y, d = e.x >> 8;
        if ((unsigned)state[idx] <= d) continue;
        if (mode == 6 && d > best) continue;
        const int oct = (int)(e.x & 0xFF);
        if (d < best) {
            second = best;
            second_level = best_level;
            best = d;
            best_level = oct;
            best_idx = (int)idx;
        } else if (track_second && d < second) {
            second_level = oct;
            second = d;
        }
    }
    *best_out = best;
    if (best_idx < 0 || best > thr) return -1;
    if (mode == 0 && best_level == second_level && (float)best > __fmul_rn(lowe_ratio, (float)second)) return -1;
    if (mode >= 4 && __fmul_rn((float)second, lowe_ratio) < (float)best) return -1;
    return best_idx;
}

// G3: one warp; shared memory: [claim per keypoint (int)][state per keypoint (u16)].  A lane's decision is safe to commit when
// no lower lane of the batch wants ANY keypoint of its list (that is the only way an earlier landmark can change a later one's
// outcome).  Mode 2 is stateless: every decision commits at once.
template <class Dev>
__global__ void __launch_bounds__(32) guided_resolve_kernel(const Dev* __restrict__ gs, int mode, unsigned thr, float lowe_ratio) {
    extern __shared__ unsigned guided_smem[];
    const Dev g = gs[blockIdx.x];
    const uint2* lists = g.lists;
    const int* list_len = g.list_len;
    unsigned char* occupied_io = g.occupied;
    int *match_out = g.match_out, *n_matches = g.n_matches, *owner = g.owner;
    const int lane = threadIdx.x;
    int* claim = reinterpret_cast<int*>(guided_smem);
    unsigned short* state = reinterpret_cast<unsigned short*>(guided_smem + g.n_train);
    for (int i = lane; i < g.n_train; i += 32) {
        claim[i] = 255;
        state[i] = mode == 4 ? (unsigned short)kMaxDist : ((occupied_io && occupied_io[i]) ? 0 : 0xFFFF);
        if (mode == 4) owner[i] = -1;
    }
    for (int q = lane; q < g.n_queries; q += 32) match_out[q] = -1;
    __syncwarp();
    int total = 0;
    for (int base = 0; base < g.n_queries; base += 32) {
        const int q = base + lane;
        const int len = (q < g.n_queries) ? list_len[q] : 0;
        const uint2* list = lists + (size_t)min(q, g.n_queries - 1) * g.cap;
        unsigned pending = __ballot_sync(0xFFFFFFFFu, len > 0);
        while (pending) {
            const bool mine = (pending >> lane) & 1u;
            unsigned best = kMaxDist;
            const int acc = mine ? guided_decide(list, len, state, mode, thr, lowe_ratio, &best) : -1;
            unsigned commit = pending;
            if (mode != 2) {
                if (acc >= 0) atomicMin(&claim[acc], lane);  // claim[idx] = lowest lane that wants idx this round
                __syncwarp();
                bool conflict = false;
                if (mine)
                    for (int k = 0; k < len; ++k) conflict |= claim[list[k].y] < lane;
                const unsigned unsafe = __ballot_sync(0xFFFFFFFFu, mine && conflict);
                if (unsafe) commit = pending & ((1u << (__ffs(unsafe) - 1)) - 1u);
                __syncwarp();
                if (acc >= 0) claim[acc] = 255;  // reset for the next round
            }
            const bool do_commit = ((commit >> lane) & 1u) && acc >= 0;
            int stolen = 0;
            if (do_commit) {
                match_out[q] = acc;
                if (mode == 4) {  // area.cc:75-87: take the keypoint over from its previous owner
                    const int prev = owner[acc];
                    if (prev >= 0) {
                        match_out[prev] = -1;
                        stolen = 1;
                    }
                    owner[acc] = q;
                    state[acc] = (unsigned short)best;
                } else if (mode != 2) {
                    // projection.cc:50-53, 163-166: a keypoint is closed to later landmarks only while the landmark it carries
                    // has_observation(); a temporal landmark (no observation yet) can be overwritten by a later one
                    if (!g.q_valid || (g.q_valid[q] & 2)) state[acc] = 0;
                }
            }
            total += __popc(__ballot_sync(0xFFFFFFFFu, do_commit)) - __popc(__ballot_sync(0xFFFFFFFFu, stolen));
            pending &= ~commit;
            __syncwarp();
        }
    }
    __syncwarp();
    if (mode == 0 || mode == 1 || mode == 3)
        for (int i = lane; i < g.n_train; i += 32) occupied_io[i] = state[i] == 0;
    if (lane == 0) *n_matches = total;
}


// b200_track_local_map: the keypoint count of a frame is known on the device only (the extractor's counter)
__global__ void track_set_counts_kernel(GuidedDev* __restrict__ gs, const chain::TrackFrameDev* __restrict__ frames, int n) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f < n) gs[f].n_train = frames[f].status[0];
}

// ---- b200_motion_based_track (frame_tracker.cc:20-59) --------------------------------------------------------------------------------
// per-frame status words: [0] matches of the first search, [1] retried, [2] matches of the search that decided, [3] n_valid, [4] tracked
constexpr int kMotionStat = 8;

// One CTA per frame, after the first search: frame_tracker.cc:32-36 decides on the device whether the frame searches again.  The second
// problem shares the grid, the query arrays and the candidate scratch of the first; it has its own occupancy (a frame without landmarks:
// erase_landmarks), match_out and count.  (2 * margin) * scale_factors[l] = 2 * (margin * scale_factors[l]) exactly in float.
__global__ void __launch_bounds__(128) motion_retry_kernel(const GuidedDev* __restrict__ g1, GuidedDev* __restrict__ g2,
                                                           const chain::TrackFrameDev* __restrict__ frames, unsigned thr, int* __restrict__ stat) {
    const int f = blockIdx.x;
    const GuidedDev& a = g1[f];
    const int n_first = *a.n_matches;
    const bool retry = (unsigned)n_first < thr;
    unsigned char* occ = g2[f].occupied;
    if (threadIdx.x == 0) {
        g2[f].n_train = a.n_train;
        g2[f].n_queries = retry ? a.n_queries : 0;
        stat[kMotionStat * f] = n_first;
        stat[kMotionStat * f + 1] = retry ? 1 : 0;
    }
    if (!retry) return;
    float* margin = frames[f].q_margin;
    for (int q = threadIdx.x; q < a.n_queries; q += blockDim.x) margin[q] = __fmul_rn(2.f, margin[q]);
    for (int i = threadIdx.x; i < a.n_train; i += blockDim.x) occ[i] = 0;
}

// after the second search: the result of the search that decided becomes the frame's match_out (the second replaces the first entirely)
// and gate[f] = whether the pose optimisation runs (:38-41)
__global__ void __launch_bounds__(128) motion_select_kernel(const GuidedDev* __restrict__ g1, const GuidedDev* __restrict__ g2, unsigned thr,
                                                            int* __restrict__ stat, int* __restrict__ gate) {
    const int f = blockIdx.y;
    const bool retried = stat[kMotionStat * f + 1] != 0;
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q == 0) {
        const int n = retried ? *g2[f].n_matches : *g1[f].n_matches;
        stat[kMotionStat * f + 2] = n;
        gate[f] = (unsigned)n >= thr ? 1 : 0;
    }
    if (retried && q < g1[f].n_queries) g1[f].match_out[q] = g2[f].match_out[q];
}

// discard_outliers (frame_tracker.cc:133-150) after stage C: an outlier keypoint loses its landmark; count the keypoints that keep one
__global__ void __launch_bounds__(256) motion_discard_kernel(const chain::TrackFrameDev* __restrict__ frames, const int* __restrict__ gate, unsigned thr,
                                                             int* __restrict__ stat) {
    __shared__ int s_valid;
    const chain::TrackFrameDev& F = frames[blockIdx.x];
    if (threadIdx.x == 0) s_valid = 0;
    __syncthreads();
    const int n = F.status[0];
    int valid = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        if (F.kp_landmark_out[i] < 0) continue;
        if (F.kp_outlier[i]) F.kp_landmark_out[i] = -1;
        else ++valid;
    }
    if (valid) atomicAdd(&s_valid, valid);
    __syncthreads();
    if (threadIdx.x == 0) {
        stat[kMotionStat * blockIdx.x + 3] = s_valid;
        stat[kMotionStat * blockIdx.x + 4] = (gate[blockIdx.x] && (unsigned)s_valid >= thr) ? 1 : 0;
    }
}

// ---- b200_robust_match_based_track (frame_tracker.cc:97-131) -------------------------------------------------------------------------
// per-frame status words (stride kMotionStat, so that motion_discard_kernel writes [3] n_valid and [4] tracked): [0] brute-force matches,
// [1] essential solution valid, [2] n_inliers, [5] essential status bits
constexpr int kRobustIter = 1000;  // find_via_ransac(1000, true) (robust.cc:211)

// One CTA per frame, after the brute-force match: the essential problem of the frame's pairs (frame bearing [idx_1], keyframe bearing
// [idx_2], rows f * stride ..), its hypotheses' problem index and its run flag (n >= 5).
__global__ void __launch_bounds__(256) robust_gather_kernel(const int* __restrict__ pairs, const int* __restrict__ n_pairs, int stride,
                                                            const chain::TrackFrameDev* __restrict__ frames, const double* __restrict__ kf_bearings,
                                                            const int* __restrict__ kf_off,
                                                            double* __restrict__ b1, double* __restrict__ b2, ess::ProblemDev* __restrict__ probs,
                                                            int* __restrict__ hyp_problem) {
    const int f = blockIdx.x;
    const int n = n_pairs[f];
    const size_t row = (size_t)f * stride;
    const int* pr = pairs + 2 * row;
    const double* fb = frames[f].bearings;
    const double* kb = kf_bearings + 3 * (size_t)kf_off[f];
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int i1 = pr[2 * i], i2 = pr[2 * i + 1];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            b1[3 * (row + i) + k] = fb[3 * (size_t)i1 + k];
            b2[3 * (row + i) + k] = kb[3 * (size_t)i2 + k];
        }
    }
    for (int k = threadIdx.x; k < kRobustIter; k += blockDim.x) hyp_problem[(size_t)f * kRobustIter + k] = f;
    if (threadIdx.x == 0) probs[f] = ess::ProblemDev{n, (int)row, f * kRobustIter, kRobustIter, n >= ess::kMinSet ? 1 : 0, 1};
}

// One CTA per frame, after the RANSAC: n_inliers (0 when not valid, robust.cc:212-228), the gate n_inliers >= thr (frame_tracker.cc:105)
// and, for an applied frame, the landmark table's match_out: keyframe keypoint idx_2 -> frame keypoint idx_1 of every inlier pair
// (set_landmarks, :111).  A frame that is not applied gets no match (its buffers are not written back).
__global__ void __launch_bounds__(256) robust_apply_kernel(const int* __restrict__ pairs, const int* __restrict__ n_pairs, int stride,
                                                           const uint8_t* __restrict__ flags, const ess::ResultDev* __restrict__ results,
                                                           const chain::TrackFrameDev* __restrict__ frames, unsigned thr, int* __restrict__ stat,
                                                           int* __restrict__ gate) {
    __shared__ int s_inl;
    const int f = blockIdx.x;
    const int n = n_pairs[f];
    const size_t row = (size_t)f * stride;
    const int* pr = pairs + 2 * row;
    const bool valid = results[f].valid != 0;
    if (threadIdx.x == 0) s_inl = 0;
    int* mo = const_cast<int*>(frames[f].match_out);
    for (int q = threadIdx.x; q < frames[f].n_lm; q += blockDim.x) mo[q] = -1;
    __syncthreads();
    int c = 0;
    if (valid)
        for (int i = threadIdx.x; i < n; i += blockDim.x) c += flags[row + i] ? 1 : 0;
    if (c) atomicAdd(&s_inl, c);
    __syncthreads();
    const int n_inl = s_inl;
    const bool applied = (unsigned)n_inl >= thr;
    if (applied)
        for (int i = threadIdx.x; i < n; i += blockDim.x)
            if (flags[row + i]) mo[pr[2 * i + 1]] = pr[2 * i];
    if (threadIdx.x == 0) {
        int* st = stat + kMotionStat * f;
        st[0] = n;
        st[1] = valid ? 1 : 0;
        st[2] = n_inl;
        st[5] = results[f].status;
        gate[f] = applied ? 1 : 0;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// All-pairs matchers with greedy state other than brute_force_match:
//   match::bow_tree::match_frame_and_keyframe   src/stella_vslam/match/bow_tree.cc:169-256   (variant 0)
//   match::bow_tree::match_keyframes            bow_tree.cc:258-366                          (variant 0)
//   match::robust::match_for_triangulation      src/stella_vslam/match/robust.cc:14-146      (variant 1)
//   match::bow_tree::match_for_triangulation    bow_tree.cc:11-167                           (variant 1, with node ids)
// P1 evaluates every (row, candidate) pair once and records, per row and in candidate order, the candidates that pass the
// state-independent gates with a distance that can still influence the outcome (<= list_thr); the sequential part is then the
// same warp-batched replay as for the guided matchers (guided_resolve_kernel, modes 5 and 6).  A BoW node holds each keypoint
// exactly once and rows of different nodes never compete for a candidate, so visiting rows in index order with the gate
// node_1[i] == node_2[j] gives the merge-join's result.
// ---------------------------------------------------------------------------------------------------------------
struct PairsDev {
    int n_queries, n_train, cap;  // rows (side 1), candidates (side 2)
    const uint4 *desc1, *desc2;
    const float *angle1, *angle2;
    const unsigned char *valid1, *valid2, *stereo1, *stereo2;
    const int *node1, *node2;
    const double *bearing1, *bearing2;
    const float* scale1;
    double E[9], epi[3];
    int valid_epiplane;
    float residual_rad_thr;
    uint2* lists;
    int* list_len;
    unsigned char* occupied;  // always null: every candidate starts free
    const unsigned char* q_valid;  // always null (interface of the shared resolve kernel)
    int *match_out, *n_matches, *owner;
};

// match/base.h:67-79 in the reference's evaluation order (3x3 times 3, dot, norm; no contraction)
__device__ __forceinline__ bool epipolar_inlier(const double* __restrict__ b1, const double* __restrict__ b2, const double* E, float thr, float scale) {
    const double x = b2[0], y = b2[1], z = b2[2];
    const double e0 = __dadd_rn(__dadd_rn(__dmul_rn(E[0], x), __dmul_rn(E[1], y)), __dmul_rn(E[2], z));
    const double e1 = __dadd_rn(__dadd_rn(__dmul_rn(E[3], x), __dmul_rn(E[4], y)), __dmul_rn(E[5], z));
    const double e2 = __dadd_rn(__dadd_rn(__dmul_rn(E[6], x), __dmul_rn(E[7], y)), __dmul_rn(E[8], z));
    const double dot = __dadd_rn(__dadd_rn(__dmul_rn(e0, b1[0]), __dmul_rn(e1, b1[1])), __dmul_rn(e2, b1[2]));
    const double norm = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(e0, e0), __dmul_rn(e1, e1)), __dmul_rn(e2, e2)));
    double c = __ddiv_rn(dot, norm);
    c = fmax(-1.0, c);
    c = fmin(1.0, c);
    const double residual_rad = fabs(__dsub_rn(1.5707963267948966, acos(c)));
    return residual_rad < (double)__fmul_rn(thr, scale);
}

constexpr int kPairRows = 64, kPairChunk = 256;

__global__ void __launch_bounds__(kPairRows) pairs_candidates_kernel(const PairsDev* __restrict__ ps, int variant, unsigned list_thr,
                                                                    int check_orientation, int* __restrict__ overflow) {
    __shared__ uint4 s2[kPairChunk * 2];
    __shared__ float sa[kPairChunk];
    __shared__ int sn[kPairChunk];
    __shared__ unsigned char sv[kPairChunk];
    const PairsDev& g = ps[blockIdx.y];
    const int n1 = g.n_queries, n2 = g.n_train;
    if ((int)(blockIdx.x * kPairRows) >= n1) return;
    const int row = blockIdx.x * kPairRows + threadIdx.x;
    const bool active = row < n1 && (!g.valid1 || g.valid1[row]);
    uint4 q0 = make_uint4(0, 0, 0, 0), q1 = q0;
    float qa = 0.f;
    int qn = 0;
    bool q_stereo = false;
    if (active) {
        q0 = g.desc1[(size_t)row * 2];
        q1 = g.desc1[(size_t)row * 2 + 1];
        if (check_orientation) qa = g.angle1[row];
        if (g.node1) qn = g.node1[row];
        q_stereo = g.stereo1 && g.stereo1[row];
    }
    uint2* out = g.lists + (size_t)min(row, n1 - 1) * g.cap;
    int len = 0;
    for (int c0 = 0; c0 < n2; c0 += kPairChunk) {
        const int cn = min(kPairChunk, n2 - c0);
        __syncthreads();
        for (int t = threadIdx.x; t < cn * 2; t += blockDim.x) s2[t] = g.desc2[(size_t)c0 * 2 + t];
        for (int t = threadIdx.x; t < cn; t += blockDim.x) {
            sa[t] = check_orientation ? g.angle2[c0 + t] : 0.f;
            sn[t] = g.node2 ? g.node2[c0 + t] : 0;
            sv[t] = g.valid2 ? g.valid2[c0 + t] : 1;
        }
        __syncthreads();
        if (!active) continue;
#pragma unroll 4
        for (int j = 0; j < cn; ++j) {
            const unsigned dist = hamming256(q0, q1, s2[2 * j], s2[2 * j + 1]);
            if (dist > list_thr) continue;
            if (!sv[j] || sn[j] != qn) continue;
            if (check_orientation && orientation_rejects(qa, sa[j])) continue;
            if (variant == 1) {
                const double* b2 = g.bearing2 + (size_t)(c0 + j) * 3;
                if (g.valid_epiplane && !q_stereo && !(g.stereo2 && g.stereo2[c0 + j])) {  // robust.cc:87-98: too close to the epipole
                    const double cos_dist = __dadd_rn(__dadd_rn(__dmul_rn(g.epi[0], b2[0]), __dmul_rn(g.epi[1], b2[1])), __dmul_rn(g.epi[2], b2[2]));
                    if (0.99862953475 < cos_dist) continue;
                }
                if (!epipolar_inlier(g.bearing1 + (size_t)row * 3, b2, g.E, g.residual_rad_thr, g.scale1[row])) continue;
            }
            if (len < g.cap) out[len] = make_uint2(dist << 8, (unsigned)(c0 + j));
            ++len;
        }
    }
    if (row < n1) {
        if (len > g.cap) {
            atomicMax(overflow, len);
            len = g.cap;
        }
        g.list_len[row] = len;
    }
}

// ---- b200_bow_match_based_track (frame_tracker.cc:61-95) ---------------------------------------------------------------------------
// The frame is side 2 of its PairsDev: its keypoint count is known on the device only (the extractor's counter, copied by stage A)
__global__ void bow_set_counts_kernel(PairsDev* __restrict__ ps, const chain::TrackFrameDev* __restrict__ frames, int n) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f < n) ps[f].n_train = frames[f].status[0];
}

// After the resolve: n_keypoints_in must equal the keypoint count (kp_node has that many entries), the gate n_matches >= thr
// (frame_tracker.cc:69-72) and the status words (stride kMotionStat, so that motion_discard_kernel writes [3] n_valid and [4] tracked):
// [0] n_matches.  The resolve's match_out (keyframe keypoint -> frame keypoint) is the frame's landmark table for stage C.
__global__ void bow_gate_kernel(const PairsDev* __restrict__ ps, const chain::TrackFrameDev* __restrict__ frames, int n, unsigned thr,
                                int* __restrict__ stat, int* __restrict__ gate) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n) return;
    const chain::TrackFrameDev& F = frames[f];
    if (F.n_kp_in != F.status[0]) F.status[1] = 1;
    const int nm = *ps[f].n_matches;
    stat[kMotionStat * f] = nm;
    gate[f] = (unsigned)nm >= thr ? 1 : 0;
}

// The distances that can still matter in the BoW variant of the all-pairs matchers: the match itself needs <= 50; a second-best above
// T can no longer fail the ratio test (lowe * (T + 1) >= 50 >= best, bow_tree.cc:232-239).  Triangulation never looks above 50
// (robust.cc:83-85).
static unsigned pairs_list_thr(float lowe_ratio, bool tri) {
    unsigned list_thr = kThrLow;
    if (!tri)
        while (list_thr < 255u && lowe_ratio * (float)(list_thr + 1) < (float)kThrLow) ++list_thr;
    return list_thr;
}

// ---------------------------------------------------------------------------------------------------------------
// match::stereo  (src/stella_vslam/match/stereo.cc:20-251): row-band candidates, arg-min Hamming < 75, 11x11 L1 patch correlation
// over +-5 px on the keypoint's pyramid level, parabola sub-pixel, rejection above twice the median correlation.
// Left keypoints are independent of each other: S1 (thread per left keypoint, right keypoints streamed through shared memory),
// S2 (warp per left keypoint: patch correlation on the pyramid levels that the two extractors keep on the device),
// S3 (one CTA: exact median by two-pass radix select, then the rejection).
// ---------------------------------------------------------------------------------------------------------------
constexpr int kStereoMaxLevels = 16;
constexpr unsigned kStereoThr = (100u + 50u) / 2u;  // stereo.h:99
struct StereoLevel {
    const unsigned char *left, *right;
    unsigned long long pitch_l, pitch_r;
    int w, h;
    float sf, inv_sf;
};
struct StereoDev {
    StereoLevel lv[kStereoMaxLevels];
    int n_levels, n_left, n_right;
    const b200_keypoint_t *kl, *kr;
    const uint4 *dl, *dr;
    float fxb, max_disp;
    int* best_right;  // [n_left]
    float *x_right, *depth;
    int* corr;        // [n_left], -1 = no stereo match
    int* n_kept;
};

constexpr int kStereoRows = 64, kStereoChunk = 256;

__global__ void __launch_bounds__(kStereoRows) stereo_match_kernel(const StereoDev* __restrict__ sp) {
    __shared__ uint4 sd[kStereoChunk * 2];
    __shared__ float sx[kStereoChunk];
    __shared__ int slo[kStereoChunk], shi[kStereoChunk], soct[kStereoChunk];
    const StereoDev& g = *sp;
    const int i = blockIdx.x * kStereoRows + threadIdx.x;
    const bool active = i < g.n_left;
    uint4 q0 = make_uint4(0, 0, 0, 0), q1 = q0;
    int row = -1, level = 0;
    float min_x = 0.f, max_x = -1.f;
    if (active) {
        const b200_keypoint_t k = g.kl[i];
        q0 = g.dl[(size_t)i * 2];
        q1 = g.dl[(size_t)i * 2 + 1];
        level = k.octave;
        row = (int)k.y;                       // indices_right_in_row.at(y_left): float -> size_t truncation (stereo.cc:41)
        min_x = __fsub_rn(k.x, g.max_disp);   // stereo.cc:47-48 (min_disp_ = 0)
        max_x = k.x;
    }
    const bool searching = active && !(max_x < 0.f);
    unsigned best = make_key(kStereoThr, 0);  // only strictly smaller distances win (stereo.cc:172)
    for (int c0 = 0; c0 < g.n_right; c0 += kStereoChunk) {
        const int cn = min(kStereoChunk, g.n_right - c0);
        __syncthreads();
        for (int t = threadIdx.x; t < cn * 2; t += blockDim.x) sd[t] = g.dr[(size_t)c0 * 2 + t];
        for (int t = threadIdx.x; t < cn; t += blockDim.x) {
            const b200_keypoint_t k = g.kr[c0 + t];
            const float r = __fmul_rn(2.0f, g.lv[min(max(k.octave, 0), g.n_levels - 1)].sf);  // stereo.cc:131-135
            sx[t] = k.x;
            shi[t] = __float2int_ru(__fadd_rn(k.y, r));
            slo[t] = __float2int_rd(__fsub_rn(k.y, r));
            soct[t] = k.octave;
        }
        __syncthreads();
        if (!searching) continue;
        for (int j = 0; j < cn; ++j) {
            if (row < slo[j] || shi[j] < row) continue;
            if (soct[j] < level - 1 || soct[j] > level + 1) continue;  // stereo.cc:158-160
            if (sx[j] < min_x || max_x < sx[j]) continue;              // stereo.cc:163-166
            const unsigned key = make_key(hamming256(q0, q1, sd[2 * j], sd[2 * j + 1]), (unsigned)(c0 + j));
            if (key_dist(key) < key_dist(best)) best = key;           // first minimum in index order
        }
    }
    if (active) g.best_right[i] = (key_dist(best) < kStereoThr) ? (int)key_idx(best) : -1;
}

__global__ void __launch_bounds__(128) stereo_subpixel_kernel(const StereoDev* __restrict__ sp) {
    const StereoDev& g = *sp;
    const int i = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (i >= g.n_left) return;
    const int j = g.best_right[i];
    float out_x = -1.f, out_depth = -1.f;
    int out_corr = -1;
    if (j >= 0) {
        const b200_keypoint_t kl = g.kl[i];
        const StereoLevel& L = g.lv[min(max(kl.octave, 0), g.n_levels - 1)];
        const float x_right = g.kr[j].x;
        const int sxl = __float2int_rn(__fmul_rn(kl.x, L.inv_sf)), syl = __float2int_rn(__fmul_rn(kl.y, L.inv_sf));
        const int sxr = __float2int_rn(__fmul_rn(x_right, L.inv_sf));
        constexpr int win = 5, slide = 5;
        const bool in_range = !(sxr - slide - win < 0 || L.w <= sxr + slide + win);  // stereo.cc:193-197
        // the reference's rowRange/colRange would assert outside the image; the extractor's 19-px border keeps patches inside
        const bool patch_ok = sxl - win >= 0 && sxl + win < L.w && syl - win >= 0 && syl + win < L.h;
        if (in_range && patch_ok) {
            const unsigned char* pl = L.left + (size_t)syl * L.pitch_l + sxl;
            const unsigned char* pr = L.right + (size_t)syl * L.pitch_r + sxr;
            const int lc = pl[0];
            int lv[4], dyv[4], dxv[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int p = min(lane + 32 * u, 120);
                dyv[u] = p / 11 - win;
                dxv[u] = p % 11 - win;
                lv[u] = (int)pl[(long long)dyv[u] * (long long)L.pitch_l + dxv[u]] - lc;
            }
            int best_corr = 0x7FFFFFFF, best_offset = 0, c_prev = 0, c1 = 0, c2 = 0, c3 = 0;
            bool want_next = false;
            for (int off = -slide; off <= slide; ++off) {
                const int rc = pr[off];
                int s = 0;
#pragma unroll
                for (int u = 0; u < 4; ++u)
                    if (lane + 32 * u < 121) s += abs(lv[u] - ((int)pr[(long long)dyv[u] * (long long)L.pitch_r + dxv[u] + off] - rc));
                s = __reduce_add_sync(0xFFFFFFFFu, s);
                if (want_next) {
                    c3 = s;
                    want_next = false;
                }
                if (s < best_corr) {  // strict: the first minimum wins (stereo.cc:221-224)
                    best_corr = s;
                    best_offset = off;
                    c1 = c_prev;
                    c2 = s;
                    want_next = true;
                }
                c_prev = s;
            }
            if (best_offset != -slide && best_offset != slide) {
                const float f1 = (float)c1, f2 = (float)c2, f3 = (float)c3;
                const double num = (double)__fsub_rn(f1, f3);
                const double den = __dsub_rn(__dmul_rn(2.0, (double)__fadd_rn(f1, f3)), __dmul_rn(4.0, (double)f2));
                const float x_delta = __double2float_rn(__ddiv_rn(num, den));
                if (!(x_delta < -1.0f || 1.0f < x_delta)) {
                    float best_x = __fmul_rn(L.sf, __fadd_rn((float)(sxr + best_offset), x_delta));
                    float disp = __fsub_rn(kl.x, best_x);
                    if (!(disp < 0.f || g.max_disp <= disp)) {
                        if (disp <= 0.f) {  // stereo.cc:78-82
                            disp = 0.01f;
                            best_x = __fsub_rn(kl.x, disp);
                        }
                        out_depth = __fdiv_rn(g.fxb, disp);
                        out_x = best_x;
                        out_corr = best_corr;
                    }
                }
            }
        }
    }
    if (lane == 0) {
        g.x_right[i] = out_x;
        g.depth[i] = out_depth;
        g.corr[i] = out_corr;
    }
}

// exact median (element size/2 of the ascending order) of the valid correlations, then stereo.cc:96-113
__global__ void __launch_bounds__(1024) stereo_median_kernel(const StereoDev* __restrict__ sp) {
    __shared__ int hist[256];
    __shared__ int sel_hi, sel_rank, n_valid, median, n_rejected;
    const StereoDev& g = *sp;
    const int tid = threadIdx.x;
    if (tid < 256) hist[tid] = 0;
    if (tid == 0) n_valid = 0, n_rejected = 0;
    __syncthreads();
    int local = 0;
    for (int i = tid; i < g.n_left; i += blockDim.x) {
        const int c = g.corr[i];
        if (c >= 0) {
            atomicAdd(&hist[min(c >> 8, 255)], 1);  // correlations are <= 121 * 510 < 65536
            ++local;
        }
    }
    atomicAdd(&n_valid, local);
    __syncthreads();
    if (n_valid == 0) {
        if (tid == 0) *g.n_kept = 0;
        return;
    }
    if (tid == 0) {
        int k = n_valid / 2, b = 0;
        while (k >= hist[b]) k -= hist[b++];
        sel_hi = b;
        sel_rank = k;
    }
    __syncthreads();
    const int hi = sel_hi;
    __syncthreads();
    if (tid < 256) hist[tid] = 0;
    __syncthreads();
    for (int i = tid; i < g.n_left; i += blockDim.x) {
        const int c = g.corr[i];
        if (c >= 0 && min(c >> 8, 255) == hi) atomicAdd(&hist[c & 255], 1);
    }
    __syncthreads();
    if (tid == 0) {
        int k = sel_rank, b = 0;
        while (k >= hist[b]) k -= hist[b++];
        median = (hi << 8) | b;
    }
    __syncthreads();
    const float thr = __double2float_rn(__dmul_rn(2.0, (double)(float)median));
    int rejected = 0;
    for (int i = tid; i < g.n_left; i += blockDim.x) {
        const int c = g.corr[i];
        if (c >= 0 && thr < (float)c) {
            g.x_right[i] = -1.f;
            g.depth[i] = -1.f;
            ++rejected;
        }
    }
    atomicAdd(&n_rejected, rejected);
    __syncthreads();
    if (tid == 0) *g.n_kept = n_valid - n_rejected;
}

// ---------------------------------------------------------------------------------------------------------------
// data::landmark::compute_descriptor (src/stella_vslam/data/landmark.cc:199-256, SURVEY 8f N3): the representative descriptor of a
// landmark = the observation whose median Hamming distance to all observations is smallest (first index on ties).  One warp per
// landmark; row by row the lanes compute the distances into shared memory and select the element [0.5 (n - 1)] of the sorted row
// by counting (value v is the k-th smallest iff #(d < v) <= k < #(d <= v)).
// ---------------------------------------------------------------------------------------------------------------
constexpr int kLmMaxObs = 512;  // observations of one landmark handled on chip
__global__ void __launch_bounds__(128) landmark_descriptor_kernel(const uint4* __restrict__ descs, const int* __restrict__ offsets, int n_landmarks,
                                                                  int* __restrict__ best_idx_out, uint4* __restrict__ desc_out) {
    __shared__ unsigned short dist[4][kLmMaxObs];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int l = blockIdx.x * 4 + warp;
    if (l >= n_landmarks) return;
    const int o = offsets[l], n = offsets[l + 1] - o;
    if (n <= 0 || n > kLmMaxObs) {
        if (lane == 0) best_idx_out[l] = n <= 0 ? -1 : -2;  // -2: more observations than the kernel holds (reported by the host)
        return;
    }
    const int k = (int)(0.5 * (n - 1));
    unsigned best = kMaxDist;
    int best_idx = 0;
    unsigned short* d = dist[warp];
    for (int i = 0; i < n; ++i) {
        const uint4 a0 = descs[(size_t)(o + i) * 2], a1 = descs[(size_t)(o + i) * 2 + 1];
        for (int j = lane; j < n; j += 32) d[j] = (unsigned short)hamming256(a0, a1, descs[(size_t)(o + j) * 2], descs[(size_t)(o + j) * 2 + 1]);
        __syncwarp();
        unsigned med = kMaxDist + 1;
        for (int j = lane; j < n; j += 32) {
            const unsigned v = d[j];
            int lt = 0, le = 0;
            for (int t = 0; t < n; ++t) {
                const unsigned w = d[t];
                lt += w < v;
                le += w <= v;
            }
            if (lt <= k && k < le) med = min(med, v);
        }
        med = warp_min(med);
        if (med < best) {
            best = med;
            best_idx = i;
        }
        __syncwarp();
    }
    if (lane == 0) best_idx_out[l] = best_idx;
    if (desc_out && lane < 2) desc_out[(size_t)l * 2 + lane] = descs[(size_t)(o + best_idx) * 2 + lane];
}

// data::landmark::update_mean_normal_and_obs_scale_variance (src/stella_vslam/data/landmark.cc:256-311, SURVEY 8f N3): per landmark the
// normalised mean of the unit viewing directions of its observations and the ORB scale range from its reference keyframe.
// Thread per landmark; explicit round-to-nearest operations (this file is compiled with FMA contraction on).
__device__ __forceinline__ double norm3(double x, double y, double z) {
    return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)));
}
// One landmark: observed from cam_centers[3 * o_begin .. 3 * o_end), reference keyframe centre ref_center.
__device__ __forceinline__ void landmark_geometry_one(double px, double py, double pz, const double* __restrict__ cam_centers, int o_begin, int o_end,
                                                      const double* __restrict__ ref_center, float ref_scale, float inv_scale_last,
                                                      double* __restrict__ mean_normal, float& max_valid, float& min_valid) {
    double mx = 0.0, my = 0.0, mz = 0.0;
    for (int o = o_begin; o < o_end; ++o) {
        const double vx = __dsub_rn(px, cam_centers[3 * (size_t)o]), vy = __dsub_rn(py, cam_centers[3 * (size_t)o + 1]),
                     vz = __dsub_rn(pz, cam_centers[3 * (size_t)o + 2]);
        const double nrm = norm3(vx, vy, vz);
        const bool pos = nrm > 0.0;  // Eigen normalized(): unchanged when the norm is 0
        mx = __dadd_rn(mx, pos ? __ddiv_rn(vx, nrm) : vx);
        my = __dadd_rn(my, pos ? __ddiv_rn(vy, nrm) : vy);
        mz = __dadd_rn(mz, pos ? __ddiv_rn(vz, nrm) : vz);
    }
    const double mn = norm3(mx, my, mz);
    mean_normal[0] = mn > 0.0 ? __ddiv_rn(mx, mn) : mx;
    mean_normal[1] = mn > 0.0 ? __ddiv_rn(my, mn) : my;
    mean_normal[2] = mn > 0.0 ? __ddiv_rn(mz, mn) : mz;
    const double dist = norm3(__dsub_rn(px, ref_center[0]), __dsub_rn(py, ref_center[1]), __dsub_rn(pz, ref_center[2]));
    const float mxv = __double2float_rn(__dmul_rn(dist, (double)ref_scale));
    max_valid = mxv;
    min_valid = __fmul_rn(mxv, inv_scale_last);
}

__global__ void __launch_bounds__(128) landmark_geometry_kernel(int n, const double* __restrict__ pos_w, const int* __restrict__ offsets,
                                                                const double* __restrict__ cam_centers, const double* __restrict__ ref_center,
                                                                const float* __restrict__ ref_scale, float inv_scale_last,
                                                                double* __restrict__ mean_normal, float* __restrict__ max_valid,
                                                                float* __restrict__ min_valid) {
    const int l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= n) return;
    landmark_geometry_one(pos_w[3 * (size_t)l], pos_w[3 * (size_t)l + 1], pos_w[3 * (size_t)l + 2], cam_centers, offsets[l], offsets[l + 1],
                          ref_center + 3 * (size_t)l, ref_scale[l], inv_scale_last, mean_normal + 3 * (size_t)l, max_valid[l], min_valid[l]);
}

// b200_depth_landmarks: one CTA per problem.  Mode 0 sorts the (depth bits << 32 | idx) keys of the keypoints with 0 < depth in
// shared memory (positive floats order like their bit patterns, and idx breaks ties, so the order is std::sort's on pair<float,
// unsigned>); both modes then compact the walked positions with a block-wide scan so that every created landmark knows its slot.
struct DepthLmDev {
    int mode, n, n_valid, npow;  // n_valid / npow: mode 0's key count and its power-of-two padding
    double rwc[9], twc[3];
    double fx_inv, fy_inv, cx, cy, depth_thr;
    const float *x, *y, *depth;
    const int* octave;
    const unsigned char* has_lm;  // may be null
    const float* sf;
    float inv_last;
    int* out_idx;
    double *pos_w, *mean_normal;
    float *min_valid, *max_valid;
    int* n_created;
};
constexpr int kDepthLmThreads = 512;

// exclusive prefix of `flag` over the CTA (kDepthLmThreads threads, all of them calling); *total = the sum
__device__ __forceinline__ int cta_exclusive_scan(int flag, int* s_warp, int* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned ballot = __ballot_sync(0xffffffffu, flag);
    const int in_warp = __popc(ballot & ((1u << lane) - 1u));
    if (lane == 0) s_warp[warp] = __popc(ballot);
    __syncthreads();
    if (warp == 0) {
        const int v = lane < kDepthLmThreads / 32 ? s_warp[lane] : 0;
        int inc = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, inc, d);
            if (lane >= d) inc += t;
        }
        if (lane < kDepthLmThreads / 32) s_warp[lane] = inc - v;
        if (lane == kDepthLmThreads / 32 - 1) *total = inc;
    }
    __syncthreads();
    const int r = s_warp[warp] + in_warp;
    __syncthreads();  // s_warp is reused by the next call
    return r;
}

__global__ void __launch_bounds__(kDepthLmThreads) depth_landmarks_kernel(const DepthLmDev* __restrict__ probs) {
    extern __shared__ unsigned long long s_keys[];
    __shared__ int s_warp[32];
    __shared__ int s_total, s_fill, s_le;
    const DepthLmDev& P = probs[blockIdx.x];
    if (P.n_created == nullptr) return;  // the host rejected this problem
    const int tid = threadIdx.x;
    int walk;  // positions walked: sorted keys (mode 0) or keypoint indices (mode 1)
    if (P.mode == 0) {
        if (tid == 0) s_fill = s_le = 0;
        __syncthreads();
        for (int i = tid; i < P.n; i += kDepthLmThreads) {
            const float d = P.depth[i];
            if (0.f < d) {
                s_keys[atomicAdd(&s_fill, 1)] = ((unsigned long long)__float_as_uint(d) << 32) | (unsigned)i;
                if (!(P.depth_thr < (double)d)) atomicAdd(&s_le, 1);
            }
        }
        __syncthreads();
        for (int i = P.n_valid + tid; i < P.npow; i += kDepthLmThreads) s_keys[i] = ~0ull;
        __syncthreads();
        for (int k = 2; k <= P.npow; k <<= 1)  // bitonic sort, ascending
            for (int j = k >> 1; j > 0; j >>= 1) {
                for (int i = tid; i < P.npow; i += kDepthLmThreads) {
                    const int ixj = i ^ j;
                    if (ixj > i) {
                        const unsigned long long a = s_keys[i], b = s_keys[ixj];
                        if ((a > b) == ((i & k) == 0)) {
                            s_keys[i] = b;
                            s_keys[ixj] = a;
                        }
                    }
                }
                __syncthreads();
            }
        // keyframe_inserter.cc:187-191: stop at the first count with 100 < count && depth_thr < depth.  The depths ascend, so the keys
        // with depth <= depth_thr are a prefix of s_le entries and the walk covers max(101, s_le) of them.
        walk = min(P.n_valid, max(101, s_le));
    } else {
        walk = P.n;
    }
    int base_out = 0;
    for (int p0 = 0; p0 < walk; p0 += kDepthLmThreads) {
        const int p = p0 + tid;
        int idx = -1;
        if (p < walk) {
            if (P.mode == 0) {
                idx = (int)(unsigned)(s_keys[p] & 0xffffffffull);
                if (P.has_lm && P.has_lm[idx]) idx = -1;  // keyframe_inserter.cc:194-200: skipped, count still advances
            } else if (0.f < P.depth[p]) {
                idx = p;
            }
        }
        const int slot = base_out + cta_exclusive_scan(idx >= 0, s_warp, &s_total);
        base_out += s_total;
        if (idx < 0) continue;
        // data::triangulate_stereo (data/common.cc:203-214): float x, y, depth; double cx_, fx_inv_
        const double z = (double)P.depth[idx];
        const double pc0 = (double)__double2float_rn(__dmul_rn(__dmul_rn(__dsub_rn((double)P.x[idx], P.cx), z), P.fx_inv));
        const double pc1 = (double)__double2float_rn(__dmul_rn(__dmul_rn(__dsub_rn((double)P.y[idx], P.cy), z), P.fy_inv));
        double pw[3];
#pragma unroll
        for (int r = 0; r < 3; ++r)
            pw[r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(P.rwc[3 * r], pc0), __dmul_rn(P.rwc[3 * r + 1], pc1)), __dmul_rn(P.rwc[3 * r + 2], z)), P.twc[r]);
        P.out_idx[slot] = idx;
        P.pos_w[3 * (size_t)slot] = pw[0];
        P.pos_w[3 * (size_t)slot + 1] = pw[1];
        P.pos_w[3 * (size_t)slot + 2] = pw[2];
        landmark_geometry_one(pw[0], pw[1], pw[2], P.twc, 0, 1, P.twc, P.sf[P.octave[idx]], P.inv_last, P.mean_normal + 3 * (size_t)slot,
                              P.max_valid[slot], P.min_valid[slot]);
    }
    if (tid == 0) *P.n_created = base_out;
}

// b200_remove_redundant_keyframes: one CTA per problem walks the ranks in order.  The live landmark state (weighted observation
// count, observation count, per-observation erased flag) sits in device scratch owned by that CTA; a rank's erasure pass writes it
// and __syncthreads publishes it to the next rank's counting pass.  It is read with __ldcg so that no thread sees an L1 copy older
// than another thread's atomic.  Each landmark is listed at most once per rank (checked on the host), so the erasure pass touches
// every landmark from one thread only.
struct CullKfDev {
    unsigned id;
    int is_root, n;
    const int* kp_lm;
    const float* depth;  // may be null
    double depth_thr;
    int* out;  // n_valid, n_redundant, skipped, removed
};
struct CullDev {
    unsigned cur_id;
    int n_cov, n_lm;
    double thr;
    const CullKfDev* kf;
    const int *off, *rank, *octave;
    const unsigned char* weight;
    int *live_weight, *live_count;  // scratch, n_lm each
    unsigned char* erased;          // scratch, one per observation
    int* n_removed;
};
constexpr int kCullThreads = 512;

// the observation of landmark [b, e) by rank r that is still live (the host checked that there is exactly one)
__device__ __forceinline__ int cull_own_obs(const CullDev& P, int b, int e, int r) {
    for (int j = b; j < e; ++j)
        if (P.rank[j] == r && !__ldcg(P.erased + j)) return j;
    return -1;
}

__global__ void __launch_bounds__(kCullThreads) cull_keyframes_kernel(const CullDev* __restrict__ probs) {
    __shared__ int s_warp[2][kCullThreads / 32];
    __shared__ int s_removed;
    const CullDev& P = probs[blockIdx.x];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int l = tid; l < P.n_lm; l += kCullThreads) {
        int w = 0;
        for (int j = P.off[l]; j < P.off[l + 1]; ++j) w += P.weight[j];
        P.live_weight[l] = w;
        P.live_count[l] = P.off[l + 1] - P.off[l];
    }
    for (int j = tid; j < P.off[P.n_lm]; j += kCullThreads) P.erased[j] = 0;
    int n_removed = 0;
    __syncthreads();
    for (int r = 0; r < P.n_cov; ++r) {
        const CullKfDev& K = P.kf[r];
        // local_map_cleaner.cc:83-90, unsigned as the reference
        const int skipped = K.is_root ? 1 : (K.id <= P.cur_id && P.cur_id <= K.id + 2u) ? 2 : 0;
        if (skipped) {
            if (tid == 0) K.out[2] = skipped;
            continue;
        }
        // count_redundant_observations (local_map_cleaner.cc:123-193)
        int nv = 0, nr = 0;
        for (int i = tid; i < K.n; i += kCullThreads) {
            const int l = K.kp_lm[i];
            if (l < 0 || __ldcg(P.live_count + l) == 0) continue;
            if (K.depth) {
                const float d = K.depth[i];
                if (d < 0.0 || K.depth_thr < d) continue;
            }
            ++nv;
            if (__ldcg(P.live_weight + l) <= 3) continue;
            const int b = P.off[l], e = P.off[l + 1];
            const long long octave = P.octave[cull_own_obs(P, b, e, r)];
            int better = 0;
            for (int j = b; j < e; ++j) {
                if (P.rank[j] == r || __ldcg(P.erased + j)) continue;
                if (P.octave[j] <= octave + 1 && ++better >= 3) break;
            }
            nr += better >= 3;
        }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            nv += __shfl_xor_sync(0xffffffffu, nv, d);
            nr += __shfl_xor_sync(0xffffffffu, nr, d);
        }
        if (lane == 0) {
            s_warp[0][warp] = nv;
            s_warp[1][warp] = nr;
        }
        __syncthreads();
        if (tid == 0) {
            int v = 0, red = 0;
            for (int w = 0; w < kCullThreads / 32; ++w) {
                v += s_warp[0][w];
                red += s_warp[1][w];
            }
            // local_map_cleaner.cc:99: float / float, compared as double
            const int rm = P.thr <= (double)__fdiv_rn((float)(unsigned)red, (float)(unsigned)v);
            K.out[0] = v;
            K.out[1] = red;
            K.out[3] = rm;
            s_removed = rm;
        }
        __syncthreads();
        if (!s_removed) continue;  // uniform: no thread writes s_removed before the next rank's __syncthreads
        ++n_removed;
        // keyframe::prepare_for_erasing -> landmark::erase_observation for every live landmark of the rank
        for (int i = tid; i < K.n; i += kCullThreads) {
            const int l = K.kp_lm[i];
            if (l < 0 || __ldcg(P.live_count + l) == 0) continue;
            const int j = cull_own_obs(P, P.off[l], P.off[l + 1], r);
            P.erased[j] = 1;
            atomicSub(P.live_weight + l, (int)P.weight[j]);
            atomicSub(P.live_count + l, 1);  // 0 = discarded
        }
        __syncthreads();
    }
    if (tid == 0) *P.n_removed = n_removed;
}

// The stage boundaries of one tracking chain's last call: ev[0] before the upload, ev[6] after the last kernel
struct ChainTimer {
    cudaEvent_t ev[7] = {};
    bool timed = false;
    int create() {
        for (cudaEvent_t& e : ev)
            if (!e) B200_CUDA(cudaEventCreate(&e));
        return B200_OK;
    }
    // stage 0..5: ev[stage] -> ev[stage + 1], stage 6: the whole call
    int elapsed(int stage, float* ms) const {
        if (!ms || stage < 0 || stage > 6 || !timed) return B200_ERR_INVALID;
        B200_CUDA(cudaEventElapsedTime(ms, ev[stage == 6 ? 0 : stage], ev[stage == 6 ? 6 : stage + 1]));
        return B200_OK;
    }
    void destroy() {
        for (cudaEvent_t e : ev)
            if (e) cudaEventDestroy(e);
    }
};
// The index of each chain's timer in Matcher::chain_timers
enum ChainId { kLocalMapChain, kMotionChain, kRobustChain, kBowChain, kChains };

struct Matcher {
    int device = 0;
    cudaStream_t own_stream = nullptr, stream = nullptr;
    // b200_matcher_set_async_resolve: the sequential resolve pass (64 warps on the whole chip) runs on a side
    // stream so that the caller's next kernels (the next batch's extraction) fill the idle SMs; joined by the next matcher call
    cudaStream_t side_stream = nullptr;
    cudaEvent_t ev_topk = nullptr, ev_resolved = nullptr;
    bool async_resolve = false, resolve_pending = false;
    bool timing = false;
    cudaEvent_t ev_t[3] = {nullptr, nullptr, nullptr};
    ChainTimer chain_timers[kChains];  // indexed by ChainId
    int join() {  // the main stream waits for the side stream's resolve
        if (resolve_pending) {
            B200_CUDA(cudaStreamWaitEvent(stream, ev_resolved, 0));
            resolve_pending = false;
        }
        return B200_OK;
    }
    // scratch (grown on demand)
    unsigned* d_lists = nullptr;
    size_t lists_cap = 0;
    int* d_matched = nullptr;
    size_t matched_cap = 0;
    unsigned* d_taken = nullptr;
    size_t taken_cap = 0;
    // staging of every host-buffer entry point (each one synchronises before it returns, so they can share it)
    StagingArena arena;

    int grow(void** p, size_t* cap, size_t bytes) {
        if (bytes <= *cap) return B200_OK;
        B200_CUDA(cudaStreamSynchronize(stream));
        if (*p) B200_CUDA(cudaFree(*p));
        *p = nullptr;
        *cap = 0;
        const size_t want = bytes + bytes / 4 + 256;
        B200_CUDA(cudaMalloc(p, want));
        *cap = want;
        return B200_OK;
    }

    // on st: the matcher's stream, or the extractor's in the robust-match chain
    int run(cudaStream_t st, int n_problems, const Side& S1, const Side& S2, const void* valid2, int max_n1, int max_n2, float lowe, int check_ori,
            void* pairs, int pairs_stride, void* n_pairs, bool device_call = false) {
        if (n_problems <= 0) return B200_OK;
        if (max_n1 >= (1 << 22) - 1) {
            set_error("brute-force matcher supports < 4194304 keypoints per frame");
            return B200_ERR_INVALID;
        }
        int rc;
        if ((rc = join())) return rc;  // (the previous resolve still reads the candidate lists this call overwrites)
        max_n1 = std::max(max_n1, 1);
        if (pairs_stride < max_n1) {
            set_error("pairs_stride %d is smaller than the largest frame (%d keypoints)", pairs_stride, max_n1);
            return B200_ERR_CAPACITY;
        }
        const int taken_words = ceil_div(max_n1, 32);
        const int list_rows = std::max(1, ceil_div(max_n2, kListRowAlign)) * kListRowAlign;
        if ((rc = grow((void**)&d_lists, &lists_cap, sizeof(unsigned) * kTopK * (size_t)list_rows * n_problems))) return rc;
        if ((rc = grow((void**)&d_matched, &matched_cap, sizeof(int) * (size_t)max_n1 * n_problems))) return rc;
        if ((rc = grow((void**)&d_taken, &taken_cap, sizeof(unsigned) * (size_t)taken_words * n_problems))) return rc;
        if (timing) B200_CUDA(cudaEventRecord(ev_t[0], st));
        const float need = lowe > 0.f ? std::ceil((float)kThrLow / lowe) + 1.f : (float)kMaxDist;
        const unsigned cap = (unsigned)std::min((float)kMaxDist, std::max((float)kThrLow, need));
        B200_CUDA(cudaFuncSetAttribute(topk_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TcSmem) + 1024));
        topk_tc_kernel<<<dim3(ceil_div(std::max(max_n2, 1), kTcRows), n_problems), kTcThreads, sizeof(TcSmem) + 1024, st>>>(
            S1, S2, (const unsigned char*)valid2, check_ori, d_lists, list_rows, cap);
        if (timing) B200_CUDA(cudaEventRecord(ev_t[1], st));
        const size_t state_bytes = sizeof(unsigned) * ((size_t)taken_words + 2 * (size_t)max_n1);  // taken bitmap, idx_1 -> idx_2 table, claim table
        const size_t stage_bytes = sizeof(unsigned) * 9 * (size_t)max_n1;
        const int use_smem = (state_bytes + stage_bytes <= 200 * 1024) ? 2 : (state_bytes <= 200 * 1024 ? 1 : 0);
        const size_t rs_bytes = use_smem == 2 ? state_bytes + stage_bytes : state_bytes;
        if (use_smem && rs_bytes > 48 * 1024)
            B200_CUDA(cudaFuncSetAttribute(resolve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rs_bytes));
        cudaStream_t rs = st;
        if (async_resolve && device_call) {
            B200_CUDA(cudaEventRecord(ev_topk, st));
            B200_CUDA(cudaStreamWaitEvent(side_stream, ev_topk, 0));
            rs = side_stream;
        }
        resolve_kernel<<<n_problems, 32, use_smem ? rs_bytes : 0, rs>>>(S1, S2, (const unsigned char*)valid2, d_lists, lowe, check_ori, d_matched,
                                                                        d_taken, taken_words, list_rows, max_n1, pairs_stride, (int*)pairs,
                                                                        (int*)n_pairs, use_smem);
        B200_CUDA(cudaGetLastError());
        if (timing) B200_CUDA(cudaEventRecord(ev_t[2], rs));
        if (rs != st) {
            B200_CUDA(cudaEventRecord(ev_resolved, side_stream));
            resolve_pending = true;
        }
        return B200_OK;
    }
};

// Dynamic shared memory of guided_resolve_kernel for frames of up to n keypoints: a claim (int) and a state (u16) per keypoint
template <class Dev = GuidedDev>
static int guided_resolve_smem(const char* who, int n, size_t* bytes) {
    *bytes = (size_t)std::max(n, 1) * 6 + 16;
    if (*bytes > 200 * 1024) {
        set_error("%s: %d keypoints per frame exceed the on-chip occupancy table", who, n);
        return B200_ERR_CAPACITY;
    }
    if (*bytes > 48 * 1024)
        B200_CUDA(cudaFuncSetAttribute(guided_resolve_kernel<Dev>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)*bytes));
    return B200_OK;
}

}  // namespace match
}  // namespace b200

struct b200_matcher_s {
    b200::match::Matcher m;
};

// The host scaffold of the tracking chains (b200_track_local_map, b200_motion_based_track, b200_robust_match_based_track,
// b200_bow_match_based_track)
namespace b200 {
namespace chain {
using match::GuidedDev;

// The keypoint grid, image bounds and window bound of the chains that run the guided search
static bool search_params_valid(const b200_track_params_t& p) {
    return p.grid_cols > 0 && p.grid_rows > 0 && (long long)p.grid_cols * p.grid_rows <= (1 << 20) && p.img_bounds[1] > p.img_bounds[0]
           && p.img_bounds[3] > p.img_bounds[2] && p.max_candidates >= 0;
}

// The extractor's last batch and its stream, opened on the matcher's device
struct Extracted {
    const b200_keypoint_t* kps = nullptr;
    const unsigned char* descs = nullptr;
    const int* counts = nullptr;
    int stride = 0, batch = 0;
    cudaStream_t st = nullptr;
};

// Row-major 4x4 pose -> rot_cw row-major, then trans_cw
static void rt_of(const double* P, double* Rt) {
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) Rt[3 * r + c] = P[4 * r + c];
        Rt[9 + r] = P[4 * r + 3];
    }
}

// The per-frame blocks every chain has: its x_right and landmark-position inputs (taken by the chain among its inputs), its
// kp_landmark_out and status outputs (taken by Call::begin_outputs), stage A's products (kout among the outputs when the chain
// downloads kp_outlier) and, in the chains that run the guided search, its queries and scratch.
struct FrameBlocks {
    size_t xr = 0, pos = 0;  // taken by the chain among its inputs, staged by Call::frame_dev
    size_t klo, status, und, tx, ty, toct, occ, kout;
    bool guided = false;
    size_t qx, qy, qm, qxr, qlo, qhi, qval, cstart, citems, ccur, lists, llen, own;

    void take_stage_a(Layout& a, size_t kc, bool with_kout) {
        und = a.take(sizeof(b200_keypoint_t) * kc);
        tx = a.take(4 * kc);
        ty = a.take(4 * kc);
        toct = a.take(kc);
        occ = a.take(kc);
        if (with_kout) kout = a.take(kc);
    }
    void take_guided(Layout& a, size_t kc, size_t nl, size_t cells, int cap) {
        guided = true;
        qx = a.take(4 * nl);
        qy = a.take(4 * nl);
        qm = a.take(4 * nl);
        qxr = a.take(4 * nl);
        qlo = a.take(nl);
        qhi = a.take(nl);
        qval = a.take(nl);
        cstart = a.take(4 * (cells + 1));
        citems = a.take(4 * kc);
        ccur = a.take(4 * cells);
        lists = a.take(8 * (size_t)cap * nl);
        llen = a.take(4 * nl);
        own = a.take(4 * kc);
    }
};

// One call of a tracking chain.  It owns what every chain does alike: the argument checks and the extractor's batch (open), the
// TrackFrameDev table at offset 0 of the arena, stage C's outputs (begin_outputs), the arena and the stage timer (reserve), the common
// fields of every frame's TrackFrameDev and its initial pose (frame_dev), the upload of the inputs and the zeroing of the outputs
// (start), then stage C, motion_discard_kernel in a gated chain, the download and the synchronise (finish).  The entry point adds its
// own blocks, staging, launches (with mark(1) .. mark(4) between them) and results, in that order.
struct Call {
    const char* who;
    match::ChainId id;
    match::Matcher* m = nullptr;
    b200_lba_t opt = nullptr;
    const b200_track_params_t* p = nullptr;
    int n = 0;
    Extracted x;
    Layout a;
    size_t out_begin = 0, out_end = 0;  // inputs [0, out_begin), outputs [out_begin, out_end), then scratch
    size_t o_pose = 0, o_nvalid = 0;    // 16 doubles, one unsigned per frame
    bool gated = false;                 // the frame_tracker chains: a gate per frame decides whether stage C applies
    size_t o_stat = 0, o_gate = 0;      // kMotionStat words, one int per frame
    unsigned char *hb = nullptr, *db = nullptr;
    TrackFrameDev* hf = nullptr;        // the table in the pinned mirror
    const TrackFrameDev* df = nullptr;  // and on the device
    std::vector<const double*> poses;

    Call(const char* who, match::ChainId id) : who(who), id(id) {}
    match::ChainTimer& timer() const { return m->chain_timers[id]; }

    // B200_OK with nothing opened when n_frames is 0.  extra() is the entry point's own check of its parameters.
    template <class Extra>
    int open(b200_orb_t orb, b200_matcher_t h, b200_lba_t lba, const b200_track_params_t* prm, int n_frames, Extra extra) {
        if (!orb || !h || !lba || !prm || n_frames < 0) return B200_ERR_INVALID;
        if (n_frames == 0) return B200_OK;
        const b200_track_params_t& q = *prm;
        if (!(q.scale_factors && q.inv_level_sigma_sq && q.num_levels != 0 && q.num_levels <= 32 && camera_valid(q.cam) && q.num_trials_robust >= 0
              && q.num_trials >= 0 && q.num_each_iter >= 0 && extra())) {
            set_error("%s: invalid parameters", who);
            return B200_ERR_INVALID;
        }
        m = &h->m;
        opt = lba;
        p = prm;
        n = n_frames;
        int orb_device = 0;
        int rc = orb_results(orb, &x.kps, &x.descs, &x.counts, &x.stride, &x.batch, &x.st, &orb_device);
        if (rc) return rc;
        if (orb_device != m->device) {
            set_error("%s: extractor and matcher live on different devices", who);
            return B200_ERR_INVALID;
        }
        B200_CUDA(cudaSetDevice(m->device));
        a.take<TrackFrameDev>(n);  // at offset 0
        poses.resize(n);
        return B200_OK;
    }
    // Ends the inputs and takes the outputs every chain has, in this order: stage C's poses and inlier counts, in a gated chain the
    // status words and gates, then each frame's kp_landmark_out and status
    template <class Lay>
    void begin_outputs(std::vector<Lay>& lay, bool gate) {
        out_begin = a.end;
        o_pose = a.take(8 * 16 * (size_t)n);
        o_nvalid = a.take(4 * (size_t)n);
        gated = gate;
        if (gated) {
            o_stat = a.take(4 * match::kMotionStat * (size_t)n);
            o_gate = a.take(4 * (size_t)n);
        }
        for (FrameBlocks& B : lay) {
            B.klo = a.take(4 * (size_t)std::max(x.stride, 1));
            B.status = a.take(16);
        }
    }
    void end_outputs() { out_end = a.end; }
    int reserve() {
        int rc = m->arena.reserve(a.end, out_end, x.st);
        if (rc || (rc = timer().create())) return rc;
        hb = m->arena.h;
        db = m->arena.d;
        hf = m->arena.host<TrackFrameDev>(0);
        df = m->arena.dev<const TrackFrameDev>(0);
        return B200_OK;
    }
    // Frame f's entry of the table with the fields that every chain fills the same way.  x_right (may be null) and pos_w are the
    // caller's, staged into B.xr and B.pos; pose_cw is the initial pose of stage C.
    TrackFrameDev& frame_dev(int f, int frame, int n_kp_in, int n_lm, const float* x_right, const double* pos_w, const double* pose_cw,
                             const FrameBlocks& B) {
        m->arena.put(B.xr, x_right, 4 * (size_t)n_kp_in);
        m->arena.put(B.pos, pos_w, 24 * (size_t)n_lm);
        poses[f] = pose_cw;
        TrackFrameDev& t = hf[f];
        t = TrackFrameDev{};
        t.kps = x.kps + (size_t)frame * x.stride;
        t.n_kp = x.counts + frame;
        t.kp_cap = x.stride;
        t.n_kp_in = n_kp_in;
        t.n_lm = n_lm;
        t.kp_x_right = x_right ? (const float*)(db + B.xr) : nullptr;
        t.pos_w = (const double*)(db + B.pos);
        rt_of(pose_cw, t.Rt);
        for (int r = 0; r < 3; ++r) t.twc[r] = -(t.Rt[r] * t.Rt[9] + t.Rt[3 + r] * t.Rt[10] + t.Rt[6 + r] * t.Rt[11]);
        t.undist = (b200_keypoint_t*)(db + B.und);
        t.t_x = (float*)(db + B.tx);
        t.t_y = (float*)(db + B.ty);
        t.t_octave = db + B.toct;
        t.occupied = db + B.occ;
        t.kp_landmark_out = (int*)(db + B.klo);
        t.kp_outlier = db + B.kout;
        t.status = (int*)(db + B.status);
        if (B.guided) {
            t.q_x = (float*)(db + B.qx);
            t.q_y = (float*)(db + B.qy);
            t.q_margin = (float*)(db + B.qm);
            t.q_xr = (float*)(db + B.qxr);
            t.q_lo = (signed char*)(db + B.qlo);
            t.q_hi = (signed char*)(db + B.qhi);
            t.q_valid = db + B.qval;
        }
        return t;
    }
    // wait_matcher: the chain runs the brute-force matcher on the extractor's stream, and an earlier device-variant call on the
    // matcher's stream may still read this handle's brute-force scratch
    int start(bool wait_matcher = false) {
        int rc = m->join();
        if (rc) return rc;
        if (wait_matcher && m->stream != x.st) {
            B200_CUDA(cudaEventRecord(m->ev_topk, m->stream));
            B200_CUDA(cudaStreamWaitEvent(x.st, m->ev_topk, 0));
        }
        B200_CUDA(cudaEventRecord(timer().ev[0], x.st));
        B200_CUDA(m->arena.upload(out_begin, x.st));
        B200_CUDA(cudaMemsetAsync(db + out_begin, 0, out_end - out_begin, x.st));
        return B200_OK;
    }
    cudaError_t mark(int i) const { return cudaEventRecord(timer().ev[i], x.st); }
    // num_matches_thr: the threshold of motion_discard_kernel in a gated chain
    int finish(const TrackShared& sh, uint32_t num_matches_thr = 0) {
        int* d_gate = gated ? (int*)(db + o_gate) : nullptr;
        int rc = track_stage_c(opt, x.st, sh, df, hf, poses.data(), n, x.stride, p->num_trials_robust, p->num_trials, p->num_each_iter,
                               (double*)(db + o_pose), (unsigned*)(db + o_nvalid), timer().ev[5], d_gate);
        if (rc) return rc;
        if (gated) {
            match::motion_discard_kernel<<<n, 256, 0, x.st>>>(df, d_gate, num_matches_thr, (int*)(db + o_stat));
            B200_CUDA(cudaGetLastError());
        }
        B200_CUDA(cudaEventRecord(timer().ev[6], x.st));
        B200_CUDA(m->arena.download(out_begin, out_end, x.st));
        B200_CUDA(cudaStreamSynchronize(x.st));
        timer().timed = true;
        return B200_OK;
    }

    // After finish: the overflow word of the guided search, a window returned more keypoints than cap
    int overflow(size_t o_overflow, int cap) const {
        const int k = *reinterpret_cast<const int*>(hb + o_overflow);
        if (k <= 0) return B200_OK;
        set_error("%s: a search window returned %d keypoints, max_candidates is %d", who, k, cap);
        return B200_ERR_CAPACITY;
    }
    const int* status(const FrameBlocks& B) const { return reinterpret_cast<const int*>(hb + B.status); }
    // status[0] is frame f's keypoint count, status[1] != 0 when n_keypoints_in disagrees with it (B200_ERR_INVALID); a count
    // above kp_cap returns over_cap_rc
    int check(int f, const FrameBlocks& B, int n_keypoints_in, int kp_cap, int over_cap_rc) const {
        const int* s = status(B);
        if (!s[1] && s[0] <= kp_cap) return B200_OK;
        set_error("%s: frame %d has %d keypoints, n_keypoints_in is %d and kp_cap %d", who, f, s[0], n_keypoints_in, kp_cap);
        return s[1] ? B200_ERR_INVALID : over_cap_rc;
    }
    const int* stat(int f) const { return reinterpret_cast<const int*>(hb + o_stat) + match::kMotionStat * (size_t)f; }
    int gate(int f) const { return reinterpret_cast<const int*>(hb + o_gate)[f]; }
    // fewer than 5 edges (pose_optimizer_g2o.cc:116-118): the initial pose stays
    void pose(int f, const FrameBlocks& B, const double* pose_in, double* pose_out) const {
        std::memcpy(pose_out, status(B)[2] < 5 ? (const void*)pose_in : hb + o_pose + sizeof(double) * 16 * (size_t)f, sizeof(double) * 16);
    }
};

// A guided search of frame t's landmark table over the keypoints stage A wrote (n_train is set on the device from the extractor's
// counter).  t_angle and q_angle are null when the search has no orientation gate.
static GuidedDev guided_of(const b200_track_params_t& p, int cap, const TrackFrameDev& t, const FrameBlocks& B, unsigned char* db, int n_queries,
                           const uint4* t_desc, const uint4* q_desc, const float* t_angle, const float* q_angle, unsigned char* occupied,
                           int* match_out, int* n_matches) {
    GuidedDev g{};
    g.n_queries = n_queries;
    g.grid_cols = p.grid_cols;
    g.grid_rows = p.grid_rows;
    g.cap = cap;
    g.min_x = p.img_bounds[0]; g.max_x = p.img_bounds[1]; g.min_y = p.img_bounds[2]; g.max_y = p.img_bounds[3];
    g.t_x = t.t_x;
    g.t_y = t.t_y;
    g.t_angle = t_angle;
    g.t_x_right = t.kp_x_right;
    g.t_octave = t.t_octave;
    g.t_desc = t_desc;
    g.q_desc = q_desc;
    g.q_x = t.q_x;
    g.q_y = t.q_y;
    g.q_margin = t.q_margin;
    g.q_x_right = t.q_xr;
    g.q_angle = q_angle;
    g.q_min_level = t.q_lo;
    g.q_max_level = t.q_hi;
    g.q_valid = t.q_valid;
    g.owner = (int*)(db + B.own);
    g.cell_start = (int*)(db + B.cstart);
    g.cell_items = (int*)(db + B.citems);
    g.cell_cursor = (int*)(db + B.ccur);
    g.lists = (uint2*)(db + B.lists);
    g.list_len = (int*)(db + B.llen);
    g.occupied = occupied;
    g.match_out = match_out;
    g.n_matches = n_matches;
    return g;
}

// The by-value parameters of every chain; a kernel reads only the fields of its own chain
static TrackShared shared_of(const b200_track_params_t& p, double true_baseline) {
    TrackShared sh{};
    sh.model = p.cam.model;
    sh.fx = p.cam.fx; sh.fy = p.cam.fy; sh.cx = p.cam.cx; sh.cy = p.cam.cy;
    sh.k1 = p.cam.k1; sh.k2 = p.cam.k2; sh.p1 = p.cam.p1; sh.p2 = p.cam.p2; sh.k3 = p.cam.k3;
    sh.k4 = p.cam.k4; sh.distortion = p.cam.distortion;
    sh.cols = p.cam.cols; sh.rows = p.cam.rows;
    sh.fxb = p.focal_x_baseline;
    sh.min_x = p.img_bounds[0]; sh.max_x = p.img_bounds[1]; sh.min_y = p.img_bounds[2]; sh.max_y = p.img_bounds[3];
    sh.ray_cos_thr = p.ray_cos_thr;
    sh.log_scale_factor = p.log_scale_factor;
    sh.margin = p.margin;
    sh.delta = p.monocular ? std::sqrt(5.99146f) : std::sqrt(7.81473f);  // pose_optimizer_g2o.cc:73-88
    sh.num_levels = p.num_levels;
    for (unsigned l = 0; l < 32; ++l) {
        sh.scale_factors[l] = p.scale_factors[std::min(l, p.num_levels - 1)];
        sh.inv_level_sigma_sq[l] = p.inv_level_sigma_sq[std::min(l, p.num_levels - 1)];
    }
    sh.monocular = p.monocular ? 1 : 0;
    sh.true_baseline = true_baseline;
    return sh;
}
}  // namespace chain
}  // namespace b200

using b200::match::Side;

extern "C" {

int b200_matcher_create(int device, b200_matcher_t* out) {
    if (!out) return B200_ERR_INVALID;
    int rc = b200::require_device(device);
    if (rc) return rc;
    b200_matcher_s* h = new (std::nothrow) b200_matcher_s();
    if (!h) return B200_ERR_INVALID;
    h->m.device = device;
    cudaError_t e = cudaStreamCreateWithFlags(&h->m.own_stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&h->m.side_stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->m.ev_topk, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->m.ev_resolved, cudaEventDisableTiming);
    for (int i = 0; i < 3 && e == cudaSuccess; ++i) e = cudaEventCreate(&h->m.ev_t[i]);
    if (e != cudaSuccess) {
        delete h;
        return b200::cuda_fail(e, "stream creation", __FILE__, __LINE__);
    }
    h->m.stream = h->m.own_stream;
    *out = h;
    return B200_OK;
}

int b200_matcher_destroy(b200_matcher_t h) {
    if (!h) return B200_OK;
    cudaSetDevice(h->m.device);
    cudaStreamSynchronize(h->m.stream);
    if (h->m.side_stream) cudaStreamSynchronize(h->m.side_stream);
    cudaFree(h->m.d_lists);
    cudaFree(h->m.d_matched);
    cudaFree(h->m.d_taken);
    h->m.arena.release();
    for (int i = 0; i < 3; ++i)
        if (h->m.ev_t[i]) cudaEventDestroy(h->m.ev_t[i]);
    for (b200::match::ChainTimer& t : h->m.chain_timers) t.destroy();
    if (h->m.ev_topk) cudaEventDestroy(h->m.ev_topk);
    if (h->m.ev_resolved) cudaEventDestroy(h->m.ev_resolved);
    if (h->m.side_stream) cudaStreamDestroy(h->m.side_stream);
    if (h->m.own_stream) cudaStreamDestroy(h->m.own_stream);
    delete h;
    return B200_OK;
}

int b200_matcher_set_async_resolve(b200_matcher_t h, int enable) {
    if (!h) return B200_ERR_INVALID;
    int rc = h->m.join();
    if (rc) return rc;
    h->m.async_resolve = enable != 0;
    return B200_OK;
}

int b200_matcher_enable_timing(b200_matcher_t h, int enable) {
    if (!h) return B200_ERR_INVALID;
    h->m.timing = enable != 0;
    return B200_OK;
}

int b200_matcher_stage_ms(b200_matcher_t h, int stage, float* ms) {
    if (!h || !ms || stage < 0 || stage > 1) return B200_ERR_INVALID;
    B200_CUDA(cudaEventSynchronize(h->m.ev_t[stage + 1]));
    B200_CUDA(cudaEventElapsedTime(ms, h->m.ev_t[stage], h->m.ev_t[stage + 1]));
    return B200_OK;
}

int b200_matcher_join(b200_matcher_t h) {
    if (!h) return B200_ERR_INVALID;
    return h->m.join();
}

int b200_matcher_set_stream(b200_matcher_t h, void* stream, int use_own) {
    if (!h) return B200_ERR_INVALID;
    B200_CUDA(cudaStreamSynchronize(h->m.stream));
    if (h->m.side_stream) B200_CUDA(cudaStreamSynchronize(h->m.side_stream));
    h->m.resolve_pending = false;
    h->m.stream = use_own ? h->m.own_stream : (cudaStream_t)stream;
    return B200_OK;
}

int b200_matcher_sync(b200_matcher_t h) {
    if (!h) return B200_ERR_INVALID;
    if (h->m.resolve_pending) {
        B200_CUDA(cudaStreamSynchronize(h->m.side_stream));
        h->m.resolve_pending = false;
    }
    B200_CUDA(cudaStreamSynchronize(h->m.stream));
    return B200_OK;
}

int b200_match_bruteforce_device(b200_matcher_t h, int n_problems, const void* d_desc1, const void* d_angle1, size_t angle1_stride,
                                 const void* d_off1, const void* d_cnt1, const void* d_desc2, const void* d_angle2, size_t angle2_stride,
                                 const void* d_valid2, const void* d_off2, const void* d_cnt2, int max_n1, int max_n2, float lowe_ratio,
                                 int check_orientation, void* d_pairs, int pairs_stride, void* d_n_pairs) {
    B200_RANGE("b200:match:bruteforce_device");
    if (!h || n_problems < 0 || max_n1 < 0 || max_n2 < 0) return B200_ERR_INVALID;
    if (n_problems == 0) return B200_OK;
    if (!d_off1 || !d_off2 || !d_cnt1 || !d_cnt2 || !d_pairs || !d_n_pairs || !d_desc1 || !d_angle1 || !d_desc2 || !d_angle2) {
        b200::set_error("b200_match_bruteforce_device: null argument");
        return B200_ERR_INVALID;
    }
    B200_CUDA(cudaSetDevice(h->m.device));
    const Side S1{(const uint4*)d_desc1, (const unsigned char*)d_angle1, (long long)angle1_stride, (const int*)d_off1, (const int*)d_cnt1};
    const Side S2{(const uint4*)d_desc2, (const unsigned char*)d_angle2, (long long)angle2_stride, (const int*)d_off2, (const int*)d_cnt2};
    return h->m.run(h->m.stream, n_problems, S1, S2, d_valid2, max_n1, max_n2, lowe_ratio, check_orientation, d_pairs, pairs_stride, d_n_pairs, true);
}

int b200_match_bruteforce(b200_matcher_t h, int n_problems, const uint8_t* desc1, const void* angle1, size_t angle1_stride,
                          const int32_t* off1, const int32_t* cnt1, const uint8_t* desc2, const void* angle2, size_t angle2_stride,
                          const uint8_t* valid2, const int32_t* off2, const int32_t* cnt2, float lowe_ratio, int check_orientation,
                          int32_t* pairs, int pairs_stride, int32_t* n_pairs) {
    B200_RANGE("b200:match:bruteforce");
    if (!h || n_problems < 0) return B200_ERR_INVALID;
    if (n_problems == 0) return B200_OK;
    if (!off1 || !off2 || !cnt1 || !cnt2 || !pairs || !n_pairs || angle1_stride < sizeof(float) || angle2_stride < sizeof(float)) {
        b200::set_error("b200_match_bruteforce: null argument or angle stride < 4");
        return B200_ERR_INVALID;
    }
    auto& m = h->m;
    B200_CUDA(cudaSetDevice(m.device));
    // extents of the two sides that the problems touch
    int lo1 = INT_MAX, hi1 = 0, lo2 = INT_MAX, hi2 = 0, max_n1 = 0, max_n2 = 0;
    for (int p = 0; p < n_problems; ++p) {
        if (off1[p] < 0 || off2[p] < 0 || cnt1[p] < 0 || cnt2[p] < 0) {
            b200::set_error("b200_match_bruteforce: negative offset/count in problem %d", p);
            return B200_ERR_INVALID;
        }
        if (cnt1[p] > 0) { lo1 = std::min(lo1, off1[p]); hi1 = std::max(hi1, off1[p] + cnt1[p]); }
        if (cnt2[p] > 0) { lo2 = std::min(lo2, off2[p]); hi2 = std::max(hi2, off2[p] + cnt2[p]); }
        max_n1 = std::max(max_n1, cnt1[p]);
        max_n2 = std::max(max_n2, cnt2[p]);
    }
    if (hi1 == 0) lo1 = 0;
    if (hi2 == 0) lo2 = 0;
    const int ext1 = hi1 - lo1, ext2 = hi2 - lo2;
    if ((ext1 > 0 && (!desc1 || !angle1)) || (ext2 > 0 && (!desc2 || !angle2))) {
        b200::set_error("b200_match_bruteforce: null descriptor/angle buffer");
        return B200_ERR_INVALID;
    }
    if (pairs_stride < std::max(max_n1, 1)) {
        b200::set_error("pairs_stride %d is smaller than the largest frame (%d keypoints)", pairs_stride, max_n1);
        return B200_ERR_CAPACITY;
    }
    std::vector<int> meta(4 * (size_t)n_problems);  // off1 | cnt1 | off2 | cnt2, rebased to the staged extents
    for (int p = 0; p < n_problems; ++p) {
        meta[p] = cnt1[p] > 0 ? off1[p] - lo1 : 0;
        meta[n_problems + p] = cnt1[p];
        meta[2 * n_problems + p] = cnt2[p] > 0 ? off2[p] - lo2 : 0;
        meta[3 * n_problems + p] = cnt2[p];
    }
    // device staging, copied straight from the caller's buffers: desc1 | desc2 | angle1 | angle2 | valid2 | meta | pairs | n_pairs
    const size_t a1_bytes = ext1 > 0 ? (size_t)(ext1 - 1) * angle1_stride + sizeof(float) : 0;
    const size_t a2_bytes = ext2 > 0 ? (size_t)(ext2 - 1) * angle2_stride + sizeof(float) : 0;
    b200::Layout L;
    const size_t o_d1 = L.take((size_t)32 * ext1), o_d2 = L.take((size_t)32 * ext2), o_a1 = L.take(a1_bytes), o_a2 = L.take(a2_bytes);
    const size_t o_v2 = L.take((size_t)ext2), o_mt = L.take<int>(meta.size()), o_pr = L.take<int>(2 * (size_t)pairs_stride * n_problems);
    const size_t o_np = L.take<int>(n_problems);
    cudaStream_t st = m.stream;
    int rc = m.arena.reserve(L.end, 0, st);
    if (rc) return rc;
    unsigned char* s = m.arena.d;
    if (ext1 > 0) {
        B200_CUDA(cudaMemcpyAsync(s + o_d1, desc1 + (size_t)32 * lo1, (size_t)32 * ext1, cudaMemcpyHostToDevice, st));
        B200_CUDA(cudaMemcpyAsync(s + o_a1, (const unsigned char*)angle1 + (size_t)lo1 * angle1_stride, a1_bytes, cudaMemcpyHostToDevice, st));
    }
    if (ext2 > 0) {
        B200_CUDA(cudaMemcpyAsync(s + o_d2, desc2 + (size_t)32 * lo2, (size_t)32 * ext2, cudaMemcpyHostToDevice, st));
        B200_CUDA(cudaMemcpyAsync(s + o_a2, (const unsigned char*)angle2 + (size_t)lo2 * angle2_stride, a2_bytes, cudaMemcpyHostToDevice, st));
        if (valid2) B200_CUDA(cudaMemcpyAsync(s + o_v2, valid2 + lo2, ext2, cudaMemcpyHostToDevice, st));
    }
    B200_CUDA(cudaMemcpyAsync(s + o_mt, meta.data(), sizeof(int) * meta.size(), cudaMemcpyHostToDevice, st));
    const int* dm = (const int*)(s + o_mt);
    const Side S1{(const uint4*)(s + o_d1), s + o_a1, (long long)angle1_stride, dm, dm + n_problems};
    const Side S2{(const uint4*)(s + o_d2), s + o_a2, (long long)angle2_stride, dm + 2 * n_problems, dm + 3 * n_problems};
    rc = m.run(st, n_problems, S1, S2, valid2 ? s + o_v2 : nullptr, max_n1, max_n2, lowe_ratio, check_orientation, s + o_pr, pairs_stride,
               s + o_np);
    if (rc) return rc;
    B200_CUDA(cudaMemcpyAsync(n_pairs, s + o_np, sizeof(int) * n_problems, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaMemcpyAsync(pairs, s + o_pr, sizeof(int) * 2 * (size_t)pairs_stride * n_problems, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    return B200_OK;
}

int b200_match_guided(b200_matcher_t h, int n_problems, b200_guided_problem_t* problems, int mode, unsigned thr, float lowe_ratio,
                      int check_orientation, int max_candidates) {
    B200_RANGE("b200:match:guided");
    using b200::match::GuidedDev;
    if (!h || n_problems < 0 || mode < B200_GUIDED_LANDMARKS || mode > B200_GUIDED_AREA || max_candidates < 0) return B200_ERR_INVALID;
    if (n_problems == 0) return B200_OK;
    if (!problems) return B200_ERR_INVALID;
    auto& m = h->m;
    B200_CUDA(cudaSetDevice(m.device));
    const int cap = max_candidates ? max_candidates : 256;
    // layout of the arena: [GuidedDev x n][inputs of every problem][outputs of every problem][scratch]; the first two parts are
    // mirrored in pinned host memory and go up in one copy, the output part comes back in one copy.
    struct Lay {
        size_t tx, ty, toct, tang, txr, tdesc, qdesc, qx, qy, qm, qlo, qhi, qxr, qang, qval, qrep, sig;  // inputs
        size_t occ, mout, nm;                                                                // outputs
        size_t cstart, citems, ccur, lists, llen, own;                                       // scratch
    };
    std::vector<Lay> lay(n_problems);
    b200::Layout a;
    a.take<GuidedDev>(n_problems);  // at offset 0
    int max_q = 0, max_train = 0;
    for (int p = 0; p < n_problems; ++p) {
        const b200_guided_problem_t& P = problems[p];
        const bool need_angle = (mode == B200_GUIDED_LAST_FRAME || mode == B200_GUIDED_AREA) && check_orientation;
        const bool need_reproj = mode == B200_GUIDED_FUSE && P.do_reprojection_matching;
        const bool need_xr = P.t_x_right && (mode <= B200_GUIDED_LAST_FRAME || need_reproj);
        if (P.n_train < 0 || P.n_queries < 0 || P.grid_cols <= 0 || P.grid_rows <= 0 || !(P.max_x > P.min_x) || !(P.max_y > P.min_y)
            || (long long)P.grid_cols * P.grid_rows > (1 << 20)) {
            b200::set_error("b200_match_guided: bad sizes / image bounds in problem %d", p);
            return B200_ERR_INVALID;
        }
        if ((P.n_train > 0 && (!P.t_x || !P.t_y || !P.t_octave || !P.t_desc || (need_angle && !P.t_angle)))
            || (P.n_queries > 0
                && (!P.q_desc || !P.q_x || !P.q_y || !P.q_margin || !P.q_min_level || !P.q_max_level || !P.match_out
                    || (need_angle && !P.q_angle) || (need_xr && !P.q_x_right)
                    || (need_reproj && (!P.q_reproj || !P.inv_level_sigma_sq || P.n_levels <= 0 || P.n_levels > 256))))) {
            b200::set_error("b200_match_guided: null buffer in problem %d", p);
            return B200_ERR_INVALID;
        }
        Lay& L = lay[p];
        const size_t nt = (size_t)P.n_train, nq = (size_t)P.n_queries;
        L.tx = a.take(4 * nt);
        L.ty = a.take(4 * nt);
        L.toct = a.take(nt);
        L.tang = a.take(4 * nt);
        L.txr = a.take(4 * nt);
        L.tdesc = a.take(32 * nt);
        L.qdesc = a.take(32 * nq);
        L.qx = a.take(4 * nq);
        L.qy = a.take(4 * nq);
        L.qm = a.take(4 * nq);
        L.qlo = a.take(nq);
        L.qhi = a.take(nq);
        L.qxr = a.take(4 * nq);
        L.qang = a.take(4 * nq);
        L.qval = a.take(nq);
        L.qrep = a.take(16 * nq);
        L.sig = a.take(4 * 256);
        L.occ = a.take(nt);  // in AND out: kept at the end of the problem's input block
        max_q = std::max(max_q, P.n_queries);
        max_train = std::max(max_train, P.n_train);
    }
    const size_t in_bytes = a.end;
    const size_t out_begin = a.end;
    for (int p = 0; p < n_problems; ++p) {
        Lay& L = lay[p];
        L.mout = a.take(4 * (size_t)problems[p].n_queries);
        L.nm = a.take(4);
    }
    const size_t o_overflow = a.take(4);
    const size_t out_end = a.end;
    for (int p = 0; p < n_problems; ++p) {
        const b200_guided_problem_t& P = problems[p];
        Lay& L = lay[p];
        const size_t cells = (size_t)P.grid_cols * P.grid_rows;
        L.cstart = a.take(4 * (cells + 1));
        L.citems = a.take(4 * (size_t)P.n_train);
        L.ccur = a.take(4 * cells);
        L.lists = a.take(8 * (size_t)cap * P.n_queries);
        L.llen = a.take(4 * (size_t)P.n_queries);
        L.own = a.take(4 * (size_t)P.n_train);
    }
    size_t rs_bytes = 0;
    int rc = b200::match::guided_resolve_smem("b200_match_guided", max_train, &rs_bytes);
    if (rc) return rc;
    cudaStream_t st = m.stream;
    if ((rc = m.arena.reserve(a.end, out_end, st))) return rc;
    b200::StagingArena& A = m.arena;
    unsigned char *hb = A.h, *db = A.d;
    GuidedDev* hg = A.host<GuidedDev>(0);
    for (int p = 0; p < n_problems; ++p) {
        const b200_guided_problem_t& P = problems[p];
        const Lay& L = lay[p];
        const size_t nt = (size_t)P.n_train, nq = (size_t)P.n_queries;
        A.put(L.tx, P.t_x, 4 * nt);
        A.put(L.ty, P.t_y, 4 * nt);
        A.put(L.toct, P.t_octave, nt);
        A.put(L.tang, P.t_angle, 4 * nt);
        A.put(L.txr, P.t_x_right, 4 * nt);
        A.put(L.tdesc, P.t_desc, 32 * nt);
        A.put(L.qdesc, P.q_desc, 32 * nq);
        A.put(L.qx, P.q_x, 4 * nq);
        A.put(L.qy, P.q_y, 4 * nq);
        A.put(L.qm, P.q_margin, 4 * nq);
        A.put(L.qlo, P.q_min_level, nq);
        A.put(L.qhi, P.q_max_level, nq);
        A.put(L.qxr, P.q_x_right, 4 * nq);
        A.put(L.qang, P.q_angle, 4 * nq);
        if (P.q_valid || P.q_has_observation)  // bit 0: valid, bit 1: has_observation()
            for (int q = 0; q < nq; ++q)
                hb[L.qval + q] = (unsigned char)(((!P.q_valid || P.q_valid[q]) ? 1 : 0) | ((!P.q_has_observation || P.q_has_observation[q]) ? 2 : 0));
        const bool reproj = mode == B200_GUIDED_FUSE && P.do_reprojection_matching;
        if (reproj) {
            A.put(L.qrep, P.q_reproj, 16 * nq);
            std::memset(hb + L.sig, 0, 4 * 256);
            A.put(L.sig, P.inv_level_sigma_sq, 4 * (size_t)P.n_levels);
        }
        if (P.t_occupied && mode != B200_GUIDED_AREA) A.put(L.occ, P.t_occupied, nt);
        else std::memset(hb + L.occ, 0, nt);
        GuidedDev g{};
        g.n_train = P.n_train;
        g.n_queries = P.n_queries;
        g.grid_cols = P.grid_cols;
        g.grid_rows = P.grid_rows;
        g.cap = cap;
        g.min_x = P.min_x; g.max_x = P.max_x; g.min_y = P.min_y; g.max_y = P.max_y;
        g.t_x = (const float*)(db + L.tx);
        g.t_y = (const float*)(db + L.ty);
        g.t_angle = (const float*)(db + L.tang);
        g.t_x_right = P.t_x_right ? (const float*)(db + L.txr) : nullptr;
        g.t_octave = db + L.toct;
        g.t_desc = (const uint4*)(db + L.tdesc);
        g.q_desc = (const uint4*)(db + L.qdesc);
        g.q_x = (const float*)(db + L.qx);
        g.q_y = (const float*)(db + L.qy);
        g.q_margin = (const float*)(db + L.qm);
        g.q_x_right = (const float*)(db + L.qxr);
        g.q_angle = (const float*)(db + L.qang);
        g.q_min_level = (const signed char*)(db + L.qlo);
        g.q_max_level = (const signed char*)(db + L.qhi);
        g.q_valid = (P.q_valid || P.q_has_observation) ? db + L.qval : nullptr;
        g.q_reproj = (const double*)(db + L.qrep);
        g.inv_level_sigma_sq = (const float*)(db + L.sig);
        g.do_reproj = reproj ? 1 : 0;
        g.owner = (int*)(db + L.own);
        g.cell_start = (int*)(db + L.cstart);
        g.cell_items = (int*)(db + L.citems);
        g.cell_cursor = (int*)(db + L.ccur);
        g.lists = (uint2*)(db + L.lists);
        g.list_len = (int*)(db + L.llen);
        g.occupied = db + L.occ;
        g.match_out = (int*)(db + L.mout);
        g.n_matches = (int*)(db + L.nm);
        hg[p] = g;
    }
    B200_CUDA(A.upload(in_bytes, st));
    B200_CUDA(cudaMemsetAsync(db + o_overflow, 0, 4, st));
    const GuidedDev* dg = A.dev<const GuidedDev>(0);
    b200::match::guided_grid_kernel<<<n_problems, 1024, 0, st>>>(dg);
    b200::match::guided_candidates_kernel<<<dim3(std::max(1, b200::ceil_div(max_q, 128)), n_problems), 128, 0, st>>>(dg, mode, check_orientation,
                                                                                                                     (int*)(db + o_overflow));
    b200::match::guided_resolve_kernel<GuidedDev><<<n_problems, 32, rs_bytes, st>>>(dg, mode, thr, lowe_ratio);
    B200_CUDA(cudaGetLastError());
    // outputs: occupancy lives in the input block (copied back per problem only when asked for), the rest is contiguous
    B200_CUDA(A.download(out_begin, out_end, st));
    const bool writes_occupancy = mode == B200_GUIDED_LANDMARKS || mode == B200_GUIDED_LAST_FRAME || mode == B200_GUIDED_FUSE;
    for (int p = 0; p < n_problems; ++p)
        if (writes_occupancy && problems[p].t_occupied && problems[p].n_train > 0)
            B200_CUDA(cudaMemcpyAsync(hb + lay[p].occ, db + lay[p].occ, (size_t)problems[p].n_train, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    const int overflow = *reinterpret_cast<const int*>(hb + o_overflow);
    if (overflow > 0) {
        b200::set_error("b200_match_guided: a search window returned %d keypoints, max_candidates is %d", overflow, cap);
        return B200_ERR_CAPACITY;
    }
    for (int p = 0; p < n_problems; ++p) {
        b200_guided_problem_t& P = problems[p];
        if (P.n_queries > 0) std::memcpy(P.match_out, hb + lay[p].mout, 4 * (size_t)P.n_queries);
        P.n_matches = *reinterpret_cast<const int*>(hb + lay[p].nm);
        if (writes_occupancy && P.t_occupied && P.n_train > 0) std::memcpy(P.t_occupied, hb + lay[p].occ, (size_t)P.n_train);
    }
    return B200_OK;
}

static int chain_stage_ms(b200_matcher_t h, b200::match::ChainId id, int stage, float* ms) {
    return h ? h->m.chain_timers[id].elapsed(stage, ms) : B200_ERR_INVALID;
}
int b200_track_stage_ms(b200_matcher_t h, int stage, float* ms) { return chain_stage_ms(h, b200::match::kLocalMapChain, stage, ms); }
int b200_motion_track_stage_ms(b200_matcher_t h, int stage, float* ms) { return chain_stage_ms(h, b200::match::kMotionChain, stage, ms); }
int b200_robust_track_stage_ms(b200_matcher_t h, int stage, float* ms) { return chain_stage_ms(h, b200::match::kRobustChain, stage, ms); }
int b200_bow_track_stage_ms(b200_matcher_t h, int stage, float* ms) { return chain_stage_ms(h, b200::match::kBowChain, stage, ms); }

// The device-resident tracking chain (see include/b200vslam.h).  Arena of the matcher handle:
//   [TrackFrameDev x n][GuidedDev x n][caller inputs]                                         -- mirrored in pinned memory, one upload
//   [poses, n_valid][per frame: kp_landmark_out, status]
//   [per frame: observable, kp_outlier, match_out, n_matches][overflow]                       -- one download
//   [stage-A products, guided scratch]
int b200_track_local_map(b200_orb_t orb, b200_matcher_t h, b200_lba_t opt, const b200_track_params_t* prm, int n_frames, b200_track_frame_t* frames) {
    B200_RANGE("b200:track:local_map");
    namespace chain = b200::chain;
    using chain::TrackFrameDev;
    using b200::match::GuidedDev;
    chain::Call C("b200_track_local_map", b200::match::kLocalMapChain);
    int rc = C.open(orb, h, opt, prm, n_frames, [&] { return frames && chain::search_params_valid(*prm); });
    if (rc || n_frames == 0) return rc;
    const chain::Extracted& x = C.x;
    const int stride = x.stride;
    cudaStream_t st = x.st;
    const int cap = prm->max_candidates ? prm->max_candidates : 256;
    struct Lay : chain::FrameBlocks {
        size_t kl, nrm, lo, hi, desc, skip, hobs;  // inputs (with xr and pos)
        size_t obs, mout, nm;                      // outputs (with klo, kout and status)
    };
    std::vector<Lay> lay(n_frames);
    int max_lm = 0;
    b200::Layout& a = C.a;
    const size_t o_gd = a.take<GuidedDev>(n_frames);
    for (int f = 0; f < n_frames; ++f) {
        const b200_track_frame_t& F = frames[f];
        if (F.frame < 0 || F.frame >= x.batch || !F.pose_cw || F.n_landmarks < 0 || F.n_keypoints_in < 0 || F.kp_cap < 0
            || ((F.kp_x_right || F.kp_landmark) && F.n_keypoints_in > stride) || !F.kp_landmark_out || !F.kp_outlier
            || (F.n_landmarks > 0 && (!F.lm_pos_w || !F.lm_mean_normal || !F.lm_min_valid_dist || !F.lm_max_valid_dist || !F.lm_desc || !F.lm_observable))) {
            b200::set_error("b200_track_local_map: frame %d: bad frame index, sizes or null buffers", f);
            return B200_ERR_INVALID;
        }
        Lay& L = lay[f];
        const size_t nk = (size_t)F.n_keypoints_in, nl = (size_t)F.n_landmarks;
        L.xr = a.take(4 * nk);
        L.kl = a.take(4 * nk);
        L.pos = a.take(24 * nl);
        L.nrm = a.take(24 * nl);
        L.lo = a.take(4 * nl);
        L.hi = a.take(4 * nl);
        L.desc = a.take(32 * nl);
        L.skip = a.take(nl);
        L.hobs = a.take(nl);
        max_lm = std::max(max_lm, F.n_landmarks);
    }
    C.begin_outputs(lay, false);
    const size_t kc = (size_t)std::max(stride, 1);
    for (int f = 0; f < n_frames; ++f) {
        Lay& L = lay[f];
        const size_t nl = (size_t)frames[f].n_landmarks;
        L.obs = a.take(nl);
        L.kout = a.take(kc);
        L.mout = a.take(4 * nl);
        L.nm = a.take(4);
    }
    const size_t o_overflow = a.take(4);
    C.end_outputs();
    const size_t cells = (size_t)prm->grid_cols * prm->grid_rows;
    for (int f = 0; f < n_frames; ++f) {
        lay[f].take_stage_a(a, kc, false);
        lay[f].take_guided(a, kc, (size_t)frames[f].n_landmarks, cells, cap);
    }
    size_t rs_bytes = 0;
    if ((rc = b200::match::guided_resolve_smem(C.who, stride, &rs_bytes))) return rc;
    if ((rc = C.reserve())) return rc;
    b200::StagingArena& A = C.m->arena;
    unsigned char *hb = C.hb, *db = C.db;
    GuidedDev* hg = A.host<GuidedDev>(o_gd);
    const chain::TrackShared sh = chain::shared_of(*prm, 0.0);
    for (int f = 0; f < n_frames; ++f) {
        const b200_track_frame_t& F = frames[f];
        const Lay& L = lay[f];
        const size_t nk = (size_t)F.n_keypoints_in, nl = (size_t)F.n_landmarks;
        A.put(L.kl, F.kp_landmark, 4 * nk);
        A.put(L.nrm, F.lm_mean_normal, 24 * nl);
        A.put(L.lo, F.lm_min_valid_dist, 4 * nl);
        A.put(L.hi, F.lm_max_valid_dist, 4 * nl);
        A.put(L.desc, F.lm_desc, 32 * nl);
        A.put(L.skip, F.lm_skip, nl);
        A.put(L.hobs, F.lm_has_observation, nl);
        TrackFrameDev& t = C.frame_dev(f, F.frame, F.n_keypoints_in, F.n_landmarks, F.kp_x_right, F.lm_pos_w, F.pose_cw, L);
        t.kp_landmark = F.kp_landmark ? (const int*)(db + L.kl) : nullptr;
        t.mean_normal = (const double*)(db + L.nrm);
        t.min_d = (const float*)(db + L.lo);
        t.max_d = (const float*)(db + L.hi);
        t.lm_skip = F.lm_skip ? db + L.skip : nullptr;
        t.lm_has_obs = F.lm_has_observation ? db + L.hobs : nullptr;
        t.observable = db + L.obs;
        t.match_out = (const int*)(db + L.mout);
        hg[f] = chain::guided_of(*prm, cap, t, L, db, F.n_landmarks, reinterpret_cast<const uint4*>(x.descs + (size_t)F.frame * stride * 32),
                                 (const uint4*)(db + L.desc), nullptr, nullptr, t.occupied, (int*)(db + L.mout), (int*)(db + L.nm));
    }
    if ((rc = C.start())) return rc;
    const TrackFrameDev* df = C.df;
    GuidedDev* dg = A.dev<GuidedDev>(o_gd);
    if ((rc = chain::track_stage_a(st, sh, df, n_frames, stride, max_lm))) return rc;
    b200::match::track_set_counts_kernel<<<b200::ceil_div(n_frames, 128), 128, 0, st>>>(dg, df, n_frames);
    B200_CUDA(C.mark(1));
    b200::match::guided_grid_kernel<<<n_frames, 1024, 0, st>>>(dg);
    B200_CUDA(C.mark(2));
    b200::match::guided_candidates_kernel<<<dim3(std::max(1, b200::ceil_div(max_lm, 128)), n_frames), 128, 0, st>>>(dg, B200_GUIDED_LANDMARKS, 0,
                                                                                                                     (int*)(db + o_overflow));
    B200_CUDA(C.mark(3));
    b200::match::guided_resolve_kernel<GuidedDev><<<n_frames, 32, rs_bytes, st>>>(dg, B200_GUIDED_LANDMARKS, prm->hamming_thr, prm->lowe_ratio);
    B200_CUDA(cudaGetLastError());
    B200_CUDA(C.mark(4));
    if ((rc = C.finish(sh))) return rc;
    if ((rc = C.overflow(o_overflow, cap))) return rc;
    for (int f = 0; f < n_frames; ++f) {
        b200_track_frame_t& F = frames[f];
        const Lay& L = lay[f];
        if ((rc = C.check(f, L, F.n_keypoints_in, F.kp_cap, B200_ERR_CAPACITY))) return rc;
        const int nk = C.status(L)[0];
        F.n_keypoints = nk;
        if (F.n_landmarks > 0) std::memcpy(F.lm_observable, hb + L.obs, (size_t)F.n_landmarks);
        std::memcpy(F.kp_landmark_out, hb + L.klo, 4 * (size_t)nk);
        std::memcpy(F.kp_outlier, hb + L.kout, (size_t)nk);
        F.n_matches = *reinterpret_cast<const int*>(hb + L.nm);
        F.n_valid = reinterpret_cast<const unsigned*>(hb + C.o_nvalid)[f];
        C.pose(f, L, F.pose_cw, F.pose_cw_out);
    }
    return B200_OK;
}

// Motion-model tracking on the device (see include/b200vslam.h).  Arena of the matcher handle, as for b200_track_local_map:
//   [TrackFrameDev x n][GuidedDev x n][GuidedDev x n (second search)][caller inputs]  -- mirrored in pinned memory, one upload
//   [poses, n_valid, status words, gates][per frame: kp_landmark_out, status]
//   [per frame: match_out, n_matches][overflow]                                       -- one download
//   [stage-A products, guided scratch, second-search buffers]
int b200_motion_based_track(b200_orb_t orb, b200_matcher_t h, b200_lba_t opt, const b200_track_params_t* prm, double true_baseline,
                            uint32_t num_matches_thr, int n_frames, b200_motion_track_frame_t* frames) {
    B200_RANGE("b200:track:motion");
    namespace chain = b200::chain;
    using chain::TrackFrameDev;
    using b200::match::GuidedDev;
    chain::Call C("b200_motion_based_track", b200::match::kMotionChain);
    int rc = C.open(orb, h, opt, prm, n_frames, [&] { return frames && chain::search_params_valid(*prm) && !std::isnan(true_baseline); });
    if (rc || n_frames == 0) return rc;
    const chain::Extracted& x = C.x;
    const int stride = x.stride;
    cudaStream_t st = x.st;
    const int cap = prm->max_candidates ? prm->max_candidates : 256;
    struct Lay : chain::FrameBlocks {
        size_t desc, oct, ang, hobs;  // inputs (with xr and pos)
        size_t mout, nm;              // outputs (with klo and status)
        size_t tang;                  // stage A: keypoint angles
        size_t occ2, mout2, nm2;      // second search
    };
    std::vector<Lay> lay(n_frames);
    int max_lm = 0;
    b200::Layout& a = C.a;
    const size_t o_gd = a.take<GuidedDev>(n_frames), o_gd2 = a.take<GuidedDev>(n_frames);
    for (int f = 0; f < n_frames; ++f) {
        const b200_motion_track_frame_t& F = frames[f];
        if (F.frame < 0 || F.frame >= x.batch || !F.pose_cw || (!prm->monocular && !F.last_pose_cw) || F.n_landmarks < 0 || F.n_keypoints_in < 0
            || F.kp_cap < 0 || (F.kp_x_right && F.n_keypoints_in > stride) || !F.kp_landmark_out
            || (F.n_landmarks > 0 && (!F.lm_pos_w || !F.lm_desc || !F.lm_octave || !F.lm_angle))) {
            b200::set_error("b200_motion_based_track: frame %d: bad frame index, sizes, null buffers or no last pose", f);
            return B200_ERR_INVALID;
        }
        for (int l = 0; l < F.n_landmarks; ++l)
            if (F.lm_octave[l] >= prm->num_levels) {  // scale_factors_.at(last_scale_level) (projection.cc:159)
                b200::set_error("b200_motion_based_track: frame %d: octave %d of entry %d is not below num_levels", f, (int)F.lm_octave[l], l);
                return B200_ERR_INVALID;
            }
        Lay& L = lay[f];
        const size_t nk = (size_t)F.n_keypoints_in, nl = (size_t)F.n_landmarks;
        L.xr = a.take(4 * nk);
        L.pos = a.take(24 * nl);
        L.desc = a.take(32 * nl);
        L.oct = a.take(nl);
        L.ang = a.take(4 * nl);
        L.hobs = a.take(nl);
        max_lm = std::max(max_lm, F.n_landmarks);
    }
    C.begin_outputs(lay, true);
    const size_t kc = (size_t)std::max(stride, 1);
    for (int f = 0; f < n_frames; ++f) {
        Lay& L = lay[f];
        const size_t nl = (size_t)frames[f].n_landmarks;
        L.mout = a.take(4 * nl);
        L.nm = a.take(4);
    }
    const size_t o_overflow = a.take(4);
    C.end_outputs();
    const size_t cells = (size_t)prm->grid_cols * prm->grid_rows;
    for (int f = 0; f < n_frames; ++f) {
        Lay& L = lay[f];
        const size_t nl = (size_t)frames[f].n_landmarks;
        L.take_stage_a(a, kc, true);
        L.take_guided(a, kc, nl, cells, cap);
        L.tang = a.take(4 * kc);
        L.occ2 = a.take(kc);
        L.mout2 = a.take(4 * nl);
        L.nm2 = a.take(4);
    }
    size_t rs_bytes = 0;
    if ((rc = b200::match::guided_resolve_smem(C.who, stride, &rs_bytes))) return rc;
    if ((rc = C.reserve())) return rc;
    b200::StagingArena& A = C.m->arena;
    unsigned char* db = C.db;
    GuidedDev* hg = A.host<GuidedDev>(o_gd);
    GuidedDev* hg2 = A.host<GuidedDev>(o_gd2);
    const chain::TrackShared sh = chain::shared_of(*prm, true_baseline);
    for (int f = 0; f < n_frames; ++f) {
        const b200_motion_track_frame_t& F = frames[f];
        const Lay& L = lay[f];
        const size_t nl = (size_t)F.n_landmarks;
        A.put(L.desc, F.lm_desc, 32 * nl);
        A.put(L.oct, F.lm_octave, nl);
        A.put(L.ang, F.lm_angle, 4 * nl);
        A.put(L.hobs, F.lm_has_observation, nl);
        // kp_landmark stays null: the frame starts without landmarks (frame_tracker.cc:27)
        TrackFrameDev& t = C.frame_dev(f, F.frame, F.n_keypoints_in, F.n_landmarks, F.kp_x_right, F.lm_pos_w, F.pose_cw, L);
        t.lm_has_obs = F.lm_has_observation ? db + L.hobs : nullptr;
        t.lm_octave = db + L.oct;
        if (F.last_pose_cw) chain::rt_of(F.last_pose_cw, t.last_Rt);
        t.t_angle = (float*)(db + L.tang);
        t.match_out = (const int*)(db + L.mout);
        const uint4* t_desc = reinterpret_cast<const uint4*>(x.descs + (size_t)F.frame * stride * 32);
        const uint4* q_desc = (const uint4*)(db + L.desc);
        const float* q_angle = (const float*)(db + L.ang);
        hg[f] = chain::guided_of(*prm, cap, t, L, db, F.n_landmarks, t_desc, q_desc, t.t_angle, q_angle, t.occupied, (int*)(db + L.mout),
                                 (int*)(db + L.nm));
        // both counts of the second search are set by motion_retry_kernel
        hg2[f] = chain::guided_of(*prm, cap, t, L, db, 0, t_desc, q_desc, t.t_angle, q_angle, db + L.occ2, (int*)(db + L.mout2), (int*)(db + L.nm2));
    }
    if ((rc = C.start())) return rc;
    const TrackFrameDev* df = C.df;
    GuidedDev* dg = A.dev<GuidedDev>(o_gd);
    GuidedDev* dg2 = A.dev<GuidedDev>(o_gd2);
    int* d_stat = (int*)(db + C.o_stat);
    const unsigned thr = num_matches_thr;
    const dim3 q_grid(std::max(1, b200::ceil_div(max_lm, 128)), n_frames);
    const float lowe = 0.9f;  // projection(0.9, true): mode 1 has no ratio test
    if ((rc = chain::motion_stage_a(st, sh, df, n_frames, stride, max_lm))) return rc;
    b200::match::track_set_counts_kernel<<<b200::ceil_div(n_frames, 128), 128, 0, st>>>(dg, df, n_frames);
    B200_CUDA(C.mark(1));
    b200::match::guided_grid_kernel<<<n_frames, 1024, 0, st>>>(dg);
    B200_CUDA(C.mark(2));
    b200::match::guided_candidates_kernel<<<q_grid, 128, 0, st>>>(dg, B200_GUIDED_LAST_FRAME, 1, (int*)(db + o_overflow));
    b200::match::guided_resolve_kernel<GuidedDev><<<n_frames, 32, rs_bytes, st>>>(dg, B200_GUIDED_LAST_FRAME, prm->hamming_thr, lowe);
    B200_CUDA(C.mark(3));
    b200::match::motion_retry_kernel<<<n_frames, 128, 0, st>>>(dg, dg2, df, thr, d_stat);
    b200::match::guided_candidates_kernel<<<q_grid, 128, 0, st>>>(dg2, B200_GUIDED_LAST_FRAME, 1, (int*)(db + o_overflow));
    b200::match::guided_resolve_kernel<GuidedDev><<<n_frames, 32, rs_bytes, st>>>(dg2, B200_GUIDED_LAST_FRAME, prm->hamming_thr, lowe);
    b200::match::motion_select_kernel<<<q_grid, 128, 0, st>>>(dg, dg2, thr, d_stat, (int*)(db + C.o_gate));
    B200_CUDA(cudaGetLastError());
    B200_CUDA(C.mark(4));
    if ((rc = C.finish(sh, thr))) return rc;
    if ((rc = C.overflow(o_overflow, cap))) return rc;
    for (int f = 0; f < n_frames; ++f) {
        b200_motion_track_frame_t& F = frames[f];
        const Lay& L = lay[f];
        if ((rc = C.check(f, L, F.n_keypoints_in, F.kp_cap, B200_ERR_CAPACITY))) return rc;
        const int nk = C.status(L)[0];
        const int* ms = C.stat(f);
        F.n_keypoints = nk;
        std::memcpy(F.kp_landmark_out, C.hb + L.klo, 4 * (size_t)nk);
        F.n_matches_first = ms[0];
        F.retried = ms[1];
        F.n_matches = ms[2];
        F.n_valid = (uint32_t)ms[3];
        F.tracked = ms[4];
        C.pose(f, L, F.pose_cw, F.pose_cw_out);  // a failed frame builds no edge: the predicted pose stays
    }
    return B200_OK;
}

// Robust-match tracking on the device (see include/b200vslam.h).  Arena of the matcher handle:
//   [TrackFrameDev x n][engines][off1 | off2 | cnt2][keyframe descriptors | angles | valid | bearings, concatenated][per frame: x_right,
//   landmark positions]                                                                  -- mirrored in pinned memory, one upload
//   [poses, n_valid, status words, gates][per frame: kp_landmark_out, status]             -- one download
//   [stage-A products, pairs, essential problems and scratch]
int b200_robust_match_based_track(b200_orb_t orb, b200_matcher_t h, b200_lba_t opt, const b200_track_params_t* prm, uint32_t num_matches_thr,
                                  int n_frames, b200_robust_track_frame_t* frames) {
    B200_RANGE("b200:track:robust");
    namespace chain = b200::chain;
    using chain::TrackFrameDev;
    using b200::match::kRobustIter;
    namespace ess = b200::ess;
    chain::Call C("b200_robust_match_based_track", b200::match::kRobustChain);
    int rc = C.open(orb, h, opt, prm, n_frames, [&] { return frames && std::isfinite(prm->lowe_ratio); });
    if (rc || n_frames == 0) return rc;
    const chain::Extracted& x = C.x;
    const int stride = x.stride;
    cudaStream_t st = x.st;
    long long total_kf = 0;
    int max_kf = 0;
    for (int f = 0; f < n_frames; ++f) {
        const b200_robust_track_frame_t& F = frames[f];
        if (F.frame < 0 || F.frame >= x.batch || !F.last_pose_cw || F.n_keypoints_in < 0 || F.kp_cap < 0 || (F.kp_x_right && F.n_keypoints_in > stride)
            || !F.kp_landmark_out || F.n_kf_keypoints < 0 || (F.engine && F.engine->index > 624u)
            || (F.n_kf_keypoints > 0 && (!F.kf_desc || !F.kf_angle || !F.kf_bearings || !F.kf_valid || !F.kf_pos_w))) {
            b200::set_error("b200_robust_match_based_track: frame %d: bad frame index, sizes, engine or null buffers", f);
            return B200_ERR_INVALID;
        }
        total_kf += F.n_kf_keypoints;
        max_kf = std::max(max_kf, F.n_kf_keypoints);
    }
    if (total_kf > INT_MAX / 64 || (long long)n_frames * std::max(stride, 1) > INT_MAX / 64) {
        b200::set_error("b200_robust_match_based_track: too many keypoints in one call");
        return B200_ERR_INVALID;
    }
    const size_t kc = (size_t)std::max(stride, 1), nf = (size_t)n_frames, T2 = (size_t)std::max(total_kf, 1LL);
    const size_t NH = nf * kRobustIter, rows = nf * kc;
    struct Lay : chain::FrameBlocks {
        size_t bear, mout;  // stage A: bearings; landmark-table matches
    };
    std::vector<Lay> lay(n_frames);
    b200::Layout& a = C.a;
    const size_t o_eng = a.take<b200_mt19937_t>(n_frames);
    const size_t o_meta = a.take<int>(3 * nf);  // off1 | off2 | cnt2
    const size_t o_kdesc = a.take(32 * T2), o_kang = a.take(4 * T2), o_kval = a.take(T2), o_kbear = a.take(24 * T2);
    for (int f = 0; f < n_frames; ++f) {
        lay[f].xr = a.take(4 * (size_t)frames[f].n_keypoints_in);
        lay[f].pos = a.take(24 * (size_t)frames[f].n_kf_keypoints);
    }
    C.begin_outputs(lay, true);
    C.end_outputs();
    for (int f = 0; f < n_frames; ++f) {
        Lay& L = lay[f];
        L.take_stage_a(a, kc, true);
        L.bear = a.take(24 * kc);
        L.mout = a.take(4 * (size_t)frames[f].n_kf_keypoints);
    }
    const size_t o_cnt1 = a.take<int>(nf), o_pairs = a.take<int>(2 * rows), o_npairs = a.take<int>(nf);
    const size_t o_probs = a.take<ess::ProblemDev>(nf), o_hp = a.take<int>(NH), o_ms = a.take<int32_t>(ess::kMinSet * NH);
    const size_t o_b1 = a.take<double>(3 * rows), o_b2 = a.take<double>(3 * rows);
    const size_t o_cand = a.take<double>(9 * ess::kMaxCand * NH), o_hyp = a.take<ess::HypDev>(NH), o_sc = a.take<ess::ScoreDev>(ess::kMaxCand * NH);
    const size_t o_idx = a.take<int32_t>(rows), o_mat = a.take<double>(9 * rows), o_fl = a.take(rows), o_res = a.take<ess::ResultDev>(nf);
    if ((rc = C.reserve())) return rc;
    b200::StagingArena& A = C.m->arena;
    unsigned char* db = C.db;
    const chain::TrackShared sh = chain::shared_of(*prm, 0.0);
    int* meta = A.host<int>(o_meta);
    size_t koff = 0;
    for (int f = 0; f < n_frames; ++f) {
        const b200_robust_track_frame_t& F = frames[f];
        const Lay& L = lay[f];
        const size_t nkf = (size_t)F.n_kf_keypoints;
        if (F.engine) A.put(o_eng + sizeof(b200_mt19937_t) * f, F.engine, sizeof(b200_mt19937_t));
        else b200_mt19937_seed(A.host<b200_mt19937_t>(o_eng) + f, nullptr, 0);
        meta[f] = F.frame * stride;
        meta[n_frames + f] = (int)koff;
        meta[2 * n_frames + f] = F.n_kf_keypoints;
        A.put(o_kdesc + 32 * koff, F.kf_desc, 32 * nkf);
        A.put(o_kang + 4 * koff, F.kf_angle, 4 * nkf);
        A.put(o_kval + koff, F.kf_valid, nkf);
        A.put(o_kbear + 24 * koff, F.kf_bearings, 24 * nkf);
        koff += nkf;
        // the landmark table is the keyframe's keypoints; kp_landmark stays null: set_landmarks replaces every slot (frame_tracker.cc:111)
        TrackFrameDev& t = C.frame_dev(f, F.frame, F.n_keypoints_in, F.n_kf_keypoints, F.kp_x_right, F.kf_pos_w, F.last_pose_cw, L);
        t.match_out = (const int*)(db + L.mout);
        t.bearings = (double*)(db + L.bear);
        t.count_out = (int*)(db + o_cnt1) + f;
    }
    if ((rc = C.start(true))) return rc;
    const TrackFrameDev* df = C.df;
    const int* d_meta = A.dev<const int>(o_meta);
    int* d_pairs = (int*)(db + o_pairs);
    int* d_npairs = (int*)(db + o_npairs);
    if ((rc = chain::robust_stage_a(st, sh, df, n_frames, stride))) return rc;
    B200_CUDA(C.mark(1));
    using b200::match::Side;
    const Side S1{reinterpret_cast<const uint4*>(x.descs), reinterpret_cast<const unsigned char*>(x.kps) + offsetof(b200_keypoint_t, angle),
                  (long long)sizeof(b200_keypoint_t), d_meta, (const int*)(db + o_cnt1)};
    const Side S2{(const uint4*)(db + o_kdesc), db + o_kang, (long long)sizeof(float), d_meta + n_frames, d_meta + 2 * n_frames};
    if ((rc = C.m->run(st, n_frames, S1, S2, db + o_kval, stride, max_kf, prm->lowe_ratio, 1, d_pairs, (int)kc, d_npairs))) return rc;
    B200_CUDA(C.mark(2));
    int32_t* d_ms = (int32_t*)(db + o_ms);
    if ((rc = chain::draw_min_sets(st, n_frames, A.dev<const b200_mt19937_t>(o_eng), d_npairs, ess::kMinSet, kRobustIter, d_ms))) return rc;
    B200_CUDA(C.mark(3));
    double* d_b1 = (double*)(db + o_b1);
    double* d_b2 = (double*)(db + o_b2);
    b200::match::robust_gather_kernel<<<n_frames, 256, 0, st>>>(d_pairs, d_npairs, (int)kc, df, (const double*)(db + o_kbear), d_meta + n_frames, d_b1,
                                                                d_b2, (ess::ProblemDev*)(db + o_probs), (int*)(db + o_hp));
    B200_CUDA(cudaGetLastError());
    const ess::RansacDev rd{(const int*)(db + o_hp), (const ess::ProblemDev*)(db + o_probs), d_b1, d_b2, d_ms, (double*)(db + o_cand),
                            (ess::HypDev*)(db + o_hyp), (ess::ScoreDev*)(db + o_sc), (int32_t*)(db + o_idx), (double*)(db + o_mat), db + o_fl,
                            (ess::ResultDev*)(db + o_res)};
    if ((rc = ess::enqueue_ransac(st, n_frames, (int)NH, rd))) return rc;
    B200_CUDA(C.mark(4));
    b200::match::robust_apply_kernel<<<n_frames, 256, 0, st>>>(d_pairs, d_npairs, (int)kc, db + o_fl, (const ess::ResultDev*)(db + o_res), df,
                                                               num_matches_thr, (int*)(db + C.o_stat), (int*)(db + C.o_gate));
    B200_CUDA(cudaGetLastError());
    if ((rc = C.finish(sh, num_matches_thr))) return rc;
    for (int f = 0; f < n_frames; ++f)  // every check before the first write: an error writes nothing
        if ((rc = C.check(f, lay[f], frames[f].n_keypoints_in, frames[f].kp_cap, B200_ERR_INVALID))) return rc;
    for (int f = 0; f < n_frames; ++f) {
        b200_robust_track_frame_t& F = frames[f];
        const int nk = C.status(lay[f])[0];
        const int* rs = C.stat(f);
        F.n_keypoints = nk;
        F.n_matches = rs[0];
        F.essential_valid = rs[1];
        F.status = rs[5] ? B200_ERR_INVALID : B200_OK;
        F.n_inliers = rs[2];
        F.applied = C.gate(f);
        F.n_valid = F.applied ? (uint32_t)rs[3] : 0u;
        F.tracked = F.applied ? rs[4] : 0;
        if (!F.applied) continue;  // frame_tracker.cc:105-108: the frame is not touched
        std::memcpy(F.kp_landmark_out, C.hb + lay[f].klo, 4 * (size_t)nk);
        C.pose(f, lay[f], F.last_pose_cw, F.pose_cw_out);
    }
    return B200_OK;
}

// BoW-match tracking on the device (see include/b200vslam.h).  Arena of the matcher handle:
//   [TrackFrameDev x n][PairsDev x n][per frame: x_right, frame nodes, keyframe descriptors | angles | nodes | rows | landmark positions]
//                                                                                         -- mirrored in pinned memory, one upload
//   [poses, n_valid, status words, gates][per frame: kp_landmark_out, status][overflow]   -- one download
//   [per frame: stage-A products, angles, match_out, n_matches, candidate lists]
int b200_bow_match_based_track(b200_orb_t orb, b200_matcher_t h, b200_lba_t opt, const b200_track_params_t* prm, uint32_t num_matches_thr,
                               int n_frames, b200_bow_track_frame_t* frames) {
    B200_RANGE("b200:track:bow");
    namespace chain = b200::chain;
    using chain::TrackFrameDev;
    using b200::match::PairsDev;
    chain::Call C("b200_bow_match_based_track", b200::match::kBowChain);
    const char* who = C.who;
    int rc = C.open(orb, h, opt, prm, n_frames, [&] { return frames && std::isfinite(prm->lowe_ratio) && prm->max_candidates >= 0; });
    if (rc || n_frames == 0) return rc;
    const chain::Extracted& x = C.x;
    const int stride = x.stride;
    cudaStream_t st = x.st;
    const int cap = prm->max_candidates ? prm->max_candidates : 64;
    int max_kf = 0;
    long long list_entries = 0;
    for (int f = 0; f < n_frames; ++f) {
        const b200_bow_track_frame_t& F = frames[f];
        if (F.frame < 0 || F.frame >= x.batch || !F.last_pose_cw || F.n_keypoints_in < 0 || F.n_keypoints_in > stride || F.kp_cap < 0
            || (F.n_keypoints_in > 0 && !F.kp_node) || !F.kp_landmark_out || F.n_kf_keypoints < 0
            || (F.n_kf_keypoints > 0 && (!F.kf_desc || !F.kf_angle || !F.kf_node || !F.kf_valid || !F.kf_pos_w))) {
            b200::set_error("%s: frame %d: bad frame index, sizes or null buffers", who, f);
            return B200_ERR_INVALID;
        }
        max_kf = std::max(max_kf, F.n_kf_keypoints);
        list_entries += (long long)F.n_kf_keypoints * cap;
    }
    if (list_entries > INT_MAX || (long long)n_frames * std::max(stride, 1) > INT_MAX / 64) {
        b200::set_error("%s: too many keypoints in one call", who);
        return B200_ERR_INVALID;
    }
    const size_t kc = (size_t)std::max(stride, 1), nf = (size_t)n_frames;
    struct Lay : chain::FrameBlocks {
        size_t node, kdesc, kang, knode, kval;  // inputs (with xr and pos)
        size_t tang, mout, nm, lists, llen;     // angles of stage A; the matcher's products
    };
    std::vector<Lay> lay(n_frames);
    b200::Layout& a = C.a;
    const size_t o_pd = a.take<PairsDev>(nf);
    for (int f = 0; f < n_frames; ++f) {
        Lay& L = lay[f];
        const size_t nkf = (size_t)frames[f].n_kf_keypoints;
        L.xr = a.take(4 * (size_t)frames[f].n_keypoints_in);
        L.node = a.take(4 * kc);  // the candidate pass reads as many nodes as the extractor has keypoints
        L.kdesc = a.take(32 * nkf);
        L.kang = a.take(4 * nkf);
        L.knode = a.take(4 * nkf);
        L.kval = a.take(nkf);
        L.pos = a.take(24 * nkf);
    }
    C.begin_outputs(lay, true);
    const size_t o_overflow = a.take(4);
    C.end_outputs();
    for (int f = 0; f < n_frames; ++f) {
        Lay& L = lay[f];
        const size_t nkf = (size_t)frames[f].n_kf_keypoints;
        L.take_stage_a(a, kc, true);
        L.tang = a.take(4 * kc);
        L.mout = a.take(4 * nkf);
        L.nm = a.take(4);
        L.lists = a.take(8 * (size_t)cap * nkf);
        L.llen = a.take(4 * nkf);
    }
    size_t rs_bytes = 0;
    if ((rc = b200::match::guided_resolve_smem<PairsDev>(who, stride, &rs_bytes))) return rc;
    if ((rc = C.reserve())) return rc;
    b200::StagingArena& A = C.m->arena;
    unsigned char *hb = C.hb, *db = C.db;
    PairsDev* hp = A.host<PairsDev>(o_pd);
    const chain::TrackShared sh = chain::shared_of(*prm, 0.0);
    for (int f = 0; f < n_frames; ++f) {
        const b200_bow_track_frame_t& F = frames[f];
        const Lay& L = lay[f];
        const size_t nk = (size_t)F.n_keypoints_in, nkf = (size_t)F.n_kf_keypoints;
        A.put(L.node, F.kp_node, 4 * nk);
        A.put(L.kdesc, F.kf_desc, 32 * nkf);
        A.put(L.kang, F.kf_angle, 4 * nkf);
        A.put(L.knode, F.kf_node, 4 * nkf);
        // a keyframe keypoint takes part iff its landmark is live (bow_tree.cc:192-199) and a node lists it; a frame keypoint that no
        // node lists is then never a candidate, since only rows of its own node see it
        unsigned char* kval = hb + L.kval;
        for (size_t i = 0; i < nkf; ++i) kval[i] = (F.kf_valid[i] && F.kf_node[i] >= 0) ? 1 : 0;
        // the landmark table is the keyframe's keypoints; kp_landmark stays null: set_landmarks replaces every slot (frame_tracker.cc:75)
        TrackFrameDev& t = C.frame_dev(f, F.frame, F.n_keypoints_in, F.n_kf_keypoints, F.kp_x_right, F.kf_pos_w, F.last_pose_cw, L);
        t.t_angle = (float*)(db + L.tang);
        t.match_out = (const int*)(db + L.mout);
        PairsDev g{};
        g.n_queries = F.n_kf_keypoints;
        g.n_train = 0;  // set on the device by bow_set_counts_kernel
        g.cap = cap;
        g.desc1 = (const uint4*)(db + L.kdesc);
        g.desc2 = reinterpret_cast<const uint4*>(x.descs + (size_t)F.frame * stride * 32);
        g.angle1 = (const float*)(db + L.kang);
        g.angle2 = t.t_angle;
        g.valid1 = db + L.kval;
        g.node1 = (const int*)(db + L.knode);
        g.node2 = (const int*)(db + L.node);
        g.lists = (uint2*)(db + L.lists);
        g.list_len = (int*)(db + L.llen);
        g.match_out = (int*)(db + L.mout);
        g.n_matches = (int*)(db + L.nm);
        hp[f] = g;
    }
    if ((rc = C.start())) return rc;
    const TrackFrameDev* df = C.df;
    PairsDev* dp = A.dev<PairsDev>(o_pd);
    if ((rc = chain::track_stage_a(st, sh, df, n_frames, stride, 0))) return rc;
    b200::match::bow_set_counts_kernel<<<b200::ceil_div(n_frames, 128), 128, 0, st>>>(dp, df, n_frames);
    B200_CUDA(C.mark(1));
    b200::match::pairs_candidates_kernel<<<dim3(std::max(1, b200::ceil_div(max_kf, b200::match::kPairRows)), n_frames), b200::match::kPairRows, 0,
                                           st>>>(dp, B200_PAIRS_BOW, b200::match::pairs_list_thr(prm->lowe_ratio, false), 1, (int*)(db + o_overflow));
    B200_CUDA(C.mark(2));
    b200::match::guided_resolve_kernel<PairsDev><<<n_frames, 32, rs_bytes, st>>>(dp, 5, (unsigned)b200::match::kThrLow, prm->lowe_ratio);
    B200_CUDA(C.mark(3));
    b200::match::bow_gate_kernel<<<b200::ceil_div(n_frames, 128), 128, 0, st>>>(dp, df, n_frames, num_matches_thr, (int*)(db + C.o_stat),
                                                                                 (int*)(db + C.o_gate));
    B200_CUDA(cudaGetLastError());
    B200_CUDA(C.mark(4));
    if ((rc = C.finish(sh, num_matches_thr))) return rc;
    // every check before the first write: an error writes nothing
    for (int f = 0; f < n_frames; ++f)
        if ((rc = C.check(f, lay[f], frames[f].n_keypoints_in, frames[f].kp_cap, B200_ERR_INVALID))) return rc;
    if (*reinterpret_cast<const int*>(hb + o_overflow) > 0) {
        b200::set_error("%s: a keyframe keypoint kept %d gated candidates, max_candidates is %d", who, *reinterpret_cast<const int*>(hb + o_overflow),
                        cap);
        return B200_ERR_CAPACITY;
    }
    for (int f = 0; f < n_frames; ++f) {
        b200_bow_track_frame_t& F = frames[f];
        const int nk = C.status(lay[f])[0];
        const int* bs = C.stat(f);
        F.n_keypoints = nk;
        F.n_matches = bs[0];
        F.applied = C.gate(f);
        F.n_valid = F.applied ? (uint32_t)bs[3] : 0u;
        F.tracked = F.applied ? bs[4] : 0;
        if (!F.applied) continue;  // frame_tracker.cc:69-72: the frame is not touched
        std::memcpy(F.kp_landmark_out, hb + lay[f].klo, 4 * (size_t)nk);
        C.pose(f, lay[f], F.last_pose_cw, F.pose_cw_out);
    }
    return B200_OK;
}

int b200_match_pairs(b200_matcher_t h, int n_problems, b200_pairs_problem_t* problems, int variant, float lowe_ratio, int check_orientation,
                     int max_candidates) {
    B200_RANGE("b200:match:pairs");
    using b200::match::PairsDev;
    if (!h || n_problems < 0 || (variant != B200_PAIRS_BOW && variant != B200_PAIRS_TRIANGULATION) || max_candidates < 0) return B200_ERR_INVALID;
    if (n_problems == 0) return B200_OK;
    if (!problems) return B200_ERR_INVALID;
    auto& m = h->m;
    B200_CUDA(cudaSetDevice(m.device));
    const int cap = max_candidates ? max_candidates : 64;
    const bool tri = variant == B200_PAIRS_TRIANGULATION;
    const unsigned list_thr = b200::match::pairs_list_thr(lowe_ratio, tri);
    b200::Layout a;
    a.take<PairsDev>(n_problems);  // at offset 0
    struct Lay {
        size_t d1, a1, v1, nd1, b1, s1, st1, d2, a2, v2, nd2, b2, st2, mout, nm, lists, llen;
    };
    std::vector<Lay> lay(n_problems);
    int max_n1 = 0, max_n2 = 0;
    for (int p = 0; p < n_problems; ++p) {
        const b200_pairs_problem_t& P = problems[p];
        if (P.n1 < 0 || P.n2 < 0 || (P.n1 > 0 && (!P.desc1 || !P.match_out)) || (P.n2 > 0 && !P.desc2) || ((P.node1 == nullptr) != (P.node2 == nullptr))
            || (check_orientation && ((P.n1 > 0 && !P.angle1) || (P.n2 > 0 && !P.angle2)))
            || (tri && ((P.n1 > 0 && (!P.bearing1 || !P.scale1)) || (P.n2 > 0 && !P.bearing2)))) {
            b200::set_error("b200_match_pairs: bad sizes or null buffer in problem %d", p);
            return B200_ERR_INVALID;
        }
        Lay& L = lay[p];
        const size_t n1 = (size_t)P.n1, n2 = (size_t)P.n2;
        L.d1 = a.take(32 * n1);
        L.a1 = a.take(4 * n1);
        L.v1 = a.take(n1);
        L.nd1 = a.take(4 * n1);
        L.b1 = a.take(24 * n1);
        L.s1 = a.take(4 * n1);
        L.st1 = a.take(n1);
        L.d2 = a.take(32 * n2);
        L.a2 = a.take(4 * n2);
        L.v2 = a.take(n2);
        L.nd2 = a.take(4 * n2);
        L.b2 = a.take(24 * n2);
        L.st2 = a.take(n2);
        max_n1 = std::max(max_n1, P.n1);
        max_n2 = std::max(max_n2, P.n2);
    }
    const size_t in_bytes = a.end, out_begin = a.end;
    for (int p = 0; p < n_problems; ++p) {
        lay[p].mout = a.take(4 * (size_t)problems[p].n1);
        lay[p].nm = a.take(4);
    }
    const size_t o_overflow = a.take(4);
    const size_t out_end = a.end;
    for (int p = 0; p < n_problems; ++p) {
        lay[p].lists = a.take(8 * (size_t)cap * problems[p].n1);
        lay[p].llen = a.take(4 * (size_t)problems[p].n1);
    }
    const size_t rs_bytes = (size_t)std::max(max_n2, 1) * 6 + 16;
    if (rs_bytes > 200 * 1024) {
        b200::set_error("b200_match_pairs: %d keypoints per frame exceed the on-chip occupancy table", max_n2);
        return B200_ERR_CAPACITY;
    }
    cudaStream_t st = m.stream;
    int rc;
    if ((rc = m.arena.reserve(a.end, out_end, st))) return rc;
    b200::StagingArena& A = m.arena;
    unsigned char *hb = A.h, *db = A.d;
    PairsDev* hg = A.host<PairsDev>(0);
    for (int p = 0; p < n_problems; ++p) {
        const b200_pairs_problem_t& P = problems[p];
        const Lay& L = lay[p];
        const size_t n1 = (size_t)P.n1, n2 = (size_t)P.n2;
        A.put(L.d1, P.desc1, 32 * n1);
        A.put(L.a1, check_orientation ? P.angle1 : nullptr, 4 * n1);
        A.put(L.v1, P.valid1, n1);
        A.put(L.nd1, P.node1, 4 * n1);
        A.put(L.b1, tri ? P.bearing1 : nullptr, 24 * n1);
        A.put(L.s1, tri ? P.scale1 : nullptr, 4 * n1);
        A.put(L.st1, tri ? P.stereo1 : nullptr, n1);
        A.put(L.d2, P.desc2, 32 * n2);
        A.put(L.a2, check_orientation ? P.angle2 : nullptr, 4 * n2);
        A.put(L.v2, P.valid2, n2);
        A.put(L.nd2, P.node2, 4 * n2);
        A.put(L.b2, tri ? P.bearing2 : nullptr, 24 * n2);
        A.put(L.st2, tri ? P.stereo2 : nullptr, n2);
        PairsDev g{};
        g.n_queries = P.n1;
        g.n_train = P.n2;
        g.cap = cap;
        g.desc1 = (const uint4*)(db + L.d1);
        g.desc2 = (const uint4*)(db + L.d2);
        g.angle1 = (const float*)(db + L.a1);
        g.angle2 = (const float*)(db + L.a2);
        g.valid1 = P.valid1 ? db + L.v1 : nullptr;
        g.valid2 = P.valid2 ? db + L.v2 : nullptr;
        g.stereo1 = (tri && P.stereo1) ? db + L.st1 : nullptr;
        g.stereo2 = (tri && P.stereo2) ? db + L.st2 : nullptr;
        g.node1 = P.node1 ? (const int*)(db + L.nd1) : nullptr;
        g.node2 = P.node2 ? (const int*)(db + L.nd2) : nullptr;
        g.bearing1 = (const double*)(db + L.b1);
        g.bearing2 = (const double*)(db + L.b2);
        g.scale1 = (const float*)(db + L.s1);
        for (int k = 0; k < 9; ++k) g.E[k] = P.E_12[k];
        for (int k = 0; k < 3; ++k) g.epi[k] = P.epiplane_in_keyfrm_2[k];
        g.valid_epiplane = P.valid_epiplane;
        g.residual_rad_thr = P.residual_rad_thr;
        g.lists = (uint2*)(db + L.lists);
        g.list_len = (int*)(db + L.llen);
        g.occupied = nullptr;
        g.match_out = (int*)(db + L.mout);
        g.n_matches = (int*)(db + L.nm);
        g.owner = nullptr;
        hg[p] = g;
    }
    B200_CUDA(A.upload(in_bytes, st));
    B200_CUDA(cudaMemsetAsync(db + o_overflow, 0, 4, st));
    const PairsDev* dg = A.dev<const PairsDev>(0);
    b200::match::pairs_candidates_kernel<<<dim3(std::max(1, b200::ceil_div(max_n1, b200::match::kPairRows)), n_problems), b200::match::kPairRows, 0,
                                           st>>>(dg, variant, list_thr, check_orientation, (int*)(db + o_overflow));
    if (rs_bytes > 48 * 1024)
        B200_CUDA(cudaFuncSetAttribute(b200::match::guided_resolve_kernel<PairsDev>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rs_bytes));
    b200::match::guided_resolve_kernel<PairsDev><<<n_problems, 32, rs_bytes, st>>>(dg, tri ? 6 : 5, (unsigned)b200::match::kThrLow, lowe_ratio);
    B200_CUDA(cudaGetLastError());
    B200_CUDA(A.download(out_begin, out_end, st));
    B200_CUDA(cudaStreamSynchronize(st));
    const int overflow = *A.host<const int>(o_overflow);
    if (overflow > 0) {
        b200::set_error("b200_match_pairs: a row kept %d gated candidates, max_candidates is %d", overflow, cap);
        return B200_ERR_CAPACITY;
    }
    for (int p = 0; p < n_problems; ++p) {
        b200_pairs_problem_t& P = problems[p];
        if (P.n1 > 0) std::memcpy(P.match_out, hb + lay[p].mout, 4 * (size_t)P.n1);
        P.n_matches = *reinterpret_cast<const int*>(hb + lay[p].nm);
    }
    return B200_OK;
}

int b200_stereo_compute(b200_matcher_t h, b200_orb_t left, int frame_left, b200_orb_t right, int frame_right, const b200_keypoint_t* keypts_left,
                        const uint8_t* descs_left, int n_left, const b200_keypoint_t* keypts_right, const uint8_t* descs_right, int n_right,
                        float focal_x_baseline, float true_baseline, float* stereo_x_right, float* depths, int32_t* n_matched) {
    B200_RANGE("b200:match:stereo");
    using namespace b200::match;
    if (!h || !left || !right || n_left < 0 || n_right < 0 || (n_left > 0 && (!keypts_left || !descs_left || !stereo_x_right || !depths))
        || (n_right > 0 && (!keypts_right || !descs_right)) || !(true_baseline > 0.f)) {
        b200::set_error("b200_stereo_compute: null argument, negative count or non-positive baseline");
        return B200_ERR_INVALID;
    }
    if (n_matched) *n_matched = 0;
    if (n_left == 0) return B200_OK;
    auto& m = h->m;
    B200_CUDA(cudaSetDevice(m.device));
    StereoDev g{};
    int rc;
    for (int l = 0; l < kStereoMaxLevels; ++l) {
        int wl = 0, hl = 0, wr = 0, hr = 0;
        float sf = 0.f;
        if (b200_orb_level_info(left, l, &wl, &hl, nullptr, &sf) != B200_OK) break;
        if (b200_orb_level_info(right, l, &wr, &hr, nullptr, nullptr) != B200_OK || wl != wr || hl != hr) {
            b200::set_error("b200_stereo_compute: the two extractors hold different pyramids at level %d", l);
            return B200_ERR_INVALID;
        }
        StereoLevel& L = g.lv[l];
        size_t pl = 0, pr = 0;
        if ((rc = b200_orb_pyramid_level_view(left, frame_left, l, &L.left, &pl, &L.w, &L.h))) return rc;
        if ((rc = b200_orb_pyramid_level_view(right, frame_right, l, &L.right, &pr, nullptr, nullptr))) return rc;
        L.pitch_l = pl;
        L.pitch_r = pr;
        L.sf = sf;
        g.n_levels = l + 1;
    }
    if (g.n_levels == 0) {
        b200::set_error("b200_stereo_compute: the extractors hold no pyramid (run extract first)");
        return B200_ERR_INVALID;
    }
    // inv_scale_factors_: the float recurrence of orb_params.cc:37-48, not 1 / sf
    {
        const float inv1 = 1.0f / g.lv[g.n_levels > 1 ? 1 : 0].sf;
        g.lv[0].inv_sf = 1.0f;
        for (int l = 1; l < g.n_levels; ++l) g.lv[l].inv_sf = inv1 * g.lv[l - 1].inv_sf;
    }
    for (int i = 0; i < n_left; ++i)
        if (keypts_left[i].octave < 0 || keypts_left[i].octave >= g.n_levels) {
            b200::set_error("b200_stereo_compute: left keypoint %d has octave %d", i, keypts_left[i].octave);
            return B200_ERR_INVALID;
        }
    if ((rc = b200_orb_sync(left)) || (rc = b200_orb_sync(right))) return rc;
    b200::Layout a;
    const size_t o_g = a.take<StereoDev>(1), o_kl = a.take<b200_keypoint_t>(n_left), o_kr = a.take<b200_keypoint_t>(n_right);
    const size_t o_dl = a.take((size_t)32 * n_left), o_dr = a.take((size_t)32 * n_right);
    const size_t in_bytes = a.end, out_begin = a.end;
    const size_t o_x = a.take(4 * (size_t)n_left), o_dep = a.take(4 * (size_t)n_left), o_nk = a.take(4);
    const size_t out_end = a.end;
    const size_t o_best = a.take(4 * (size_t)n_left), o_corr = a.take(4 * (size_t)n_left);
    cudaStream_t st = m.stream;
    if ((rc = m.arena.reserve(a.end, out_end, st))) return rc;
    b200::StagingArena& A = m.arena;
    unsigned char *hb = A.h, *db = A.d;
    g.n_left = n_left;
    g.n_right = n_right;
    g.kl = (const b200_keypoint_t*)(db + o_kl);
    g.kr = (const b200_keypoint_t*)(db + o_kr);
    g.dl = (const uint4*)(db + o_dl);
    g.dr = (const uint4*)(db + o_dr);
    g.fxb = focal_x_baseline;
    g.max_disp = focal_x_baseline / true_baseline;  // stereo.cc:18
    g.best_right = (int*)(db + o_best);
    g.x_right = (float*)(db + o_x);
    g.depth = (float*)(db + o_dep);
    g.corr = (int*)(db + o_corr);
    g.n_kept = (int*)(db + o_nk);
    A.put(o_g, &g, sizeof(g));
    A.put(o_kl, keypts_left, sizeof(b200_keypoint_t) * (size_t)n_left);
    A.put(o_dl, descs_left, (size_t)32 * n_left);
    A.put(o_kr, keypts_right, sizeof(b200_keypoint_t) * (size_t)n_right);
    A.put(o_dr, descs_right, (size_t)32 * n_right);
    B200_CUDA(A.upload(in_bytes, st));
    const StereoDev* dg = A.dev<const StereoDev>(o_g);
    stereo_match_kernel<<<b200::ceil_div(n_left, kStereoRows), kStereoRows, 0, st>>>(dg);
    stereo_subpixel_kernel<<<b200::ceil_div(n_left, 4), 128, 0, st>>>(dg);
    stereo_median_kernel<<<1, 1024, 0, st>>>(dg);
    B200_CUDA(cudaGetLastError());
    B200_CUDA(A.download(out_begin, out_end, st));
    B200_CUDA(cudaStreamSynchronize(st));
    std::memcpy(stereo_x_right, hb + o_x, 4 * (size_t)n_left);
    std::memcpy(depths, hb + o_dep, 4 * (size_t)n_left);
    if (n_matched) *n_matched = *reinterpret_cast<const int*>(hb + o_nk);
    return B200_OK;
}

int b200_landmark_descriptors(b200_matcher_t h, int n_landmarks, const uint8_t* descs, const int32_t* offsets, int32_t* best_idx, uint8_t* desc_out) {
    if (!h || n_landmarks < 0) return B200_ERR_INVALID;
    if (n_landmarks == 0) return B200_OK;
    if (!offsets || !best_idx || offsets[0] != 0) {
        b200::set_error("b200_landmark_descriptors: offsets must start at 0 and best_idx must be given");
        return B200_ERR_INVALID;
    }
    for (int l = 0; l < n_landmarks; ++l)
        if (offsets[l + 1] < offsets[l]) {
            b200::set_error("b200_landmark_descriptors: offsets are not ascending at landmark %d", l);
            return B200_ERR_INVALID;
        }
    const size_t total = (size_t)offsets[n_landmarks];
    if (total > 0 && !descs) return B200_ERR_INVALID;
    auto& m = h->m;
    B200_CUDA(cudaSetDevice(m.device));
    b200::Layout a;
    const size_t o_desc = a.take(32 * total), o_off = a.take(4 * ((size_t)n_landmarks + 1));
    const size_t in_bytes = a.end, out_begin = a.end;
    const size_t o_best = a.take(4 * (size_t)n_landmarks), o_out = a.take(32 * (size_t)n_landmarks);
    const size_t out_end = a.end;
    cudaStream_t st = m.stream;
    int rc;
    if ((rc = m.arena.reserve(a.end, out_end, st))) return rc;
    b200::StagingArena& A = m.arena;
    unsigned char *hb = A.h, *db = A.d;
    A.put(o_desc, descs, 32 * total);
    A.put(o_off, offsets, 4 * ((size_t)n_landmarks + 1));
    B200_CUDA(A.upload(in_bytes, st));
    b200::match::landmark_descriptor_kernel<<<b200::ceil_div(n_landmarks, 4), 128, 0, st>>>((const uint4*)(db + o_desc), (const int*)(db + o_off), n_landmarks,
                                                                                         (int*)(db + o_best), desc_out ? (uint4*)(db + o_out) : nullptr);
    B200_CUDA(cudaGetLastError());
    B200_CUDA(A.download(out_begin, out_end, st));
    B200_CUDA(cudaStreamSynchronize(st));
    std::memcpy(best_idx, hb + o_best, 4 * (size_t)n_landmarks);
    for (int l = 0; l < n_landmarks; ++l)
        if (best_idx[l] == -2) {
            b200::set_error("b200_landmark_descriptors: landmark %d has %d observations, at most %d are supported", l, offsets[l + 1] - offsets[l],
                            b200::match::kLmMaxObs);
            return B200_ERR_CAPACITY;
        }
    if (desc_out) {
        std::memcpy(desc_out, hb + o_out, 32 * (size_t)n_landmarks);
        for (int l = 0; l < n_landmarks; ++l)
            if (best_idx[l] < 0) std::memset(desc_out + 32 * (size_t)l, 0, 32);
    }
    return B200_OK;
}

int b200_landmark_geometry(b200_matcher_t h, int n_landmarks, const double* pos_w, const int32_t* offsets, const double* cam_centers,
                           const double* ref_center, const float* ref_scale_factor, float inv_scale_factor_last, double* mean_normal,
                           float* max_valid_dist, float* min_valid_dist) {
    if (!h || n_landmarks < 0) return B200_ERR_INVALID;
    if (n_landmarks == 0) return B200_OK;
    if (!pos_w || !offsets || !ref_center || !ref_scale_factor || !mean_normal || !max_valid_dist || !min_valid_dist || offsets[0] != 0) return B200_ERR_INVALID;
    for (int l = 0; l < n_landmarks; ++l)
        if (offsets[l + 1] < offsets[l]) return B200_ERR_INVALID;
    const size_t N = (size_t)n_landmarks, total = (size_t)offsets[n_landmarks];
    if (total > 0 && !cam_centers) return B200_ERR_INVALID;
    auto& m = h->m;
    B200_CUDA(cudaSetDevice(m.device));
    b200::Layout a;
    const size_t o_p = a.take(24 * N), o_off = a.take(4 * (N + 1)), o_c = a.take(24 * total), o_r = a.take(24 * N), o_s = a.take(4 * N);
    const size_t in_bytes = a.end, out_begin = a.end;
    const size_t o_mn = a.take(24 * N), o_mx = a.take(4 * N), o_mi = a.take(4 * N);
    const size_t out_end = a.end;
    cudaStream_t st = m.stream;
    int rc;
    if ((rc = m.arena.reserve(a.end, out_end, st))) return rc;
    b200::StagingArena& A = m.arena;
    unsigned char *hb = A.h, *db = A.d;
    A.put(o_p, pos_w, 24 * N);
    A.put(o_off, offsets, 4 * (N + 1));
    A.put(o_c, cam_centers, 24 * total);
    A.put(o_r, ref_center, 24 * N);
    A.put(o_s, ref_scale_factor, 4 * N);
    B200_CUDA(A.upload(in_bytes, st));
    b200::match::landmark_geometry_kernel<<<b200::ceil_div(n_landmarks, 128), 128, 0, st>>>(n_landmarks, (const double*)(db + o_p), (const int*)(db + o_off),
                                                                                         (const double*)(db + o_c), (const double*)(db + o_r),
                                                                                         (const float*)(db + o_s), inv_scale_factor_last,
                                                                                         (double*)(db + o_mn), (float*)(db + o_mx), (float*)(db + o_mi));
    B200_CUDA(cudaGetLastError());
    B200_CUDA(A.download(out_begin, out_end, st));
    B200_CUDA(cudaStreamSynchronize(st));
    std::memcpy(mean_normal, hb + o_mn, 24 * N);
    std::memcpy(max_valid_dist, hb + o_mx, 4 * N);
    std::memcpy(min_valid_dist, hb + o_mi, 4 * N);
    return B200_OK;
}

int b200_depth_landmarks(b200_matcher_t h, int n_problems, b200_depth_landmarks_problem_t* problems) {
    B200_RANGE("b200:match:depth_landmarks");
    if (!h || n_problems < 0 || (n_problems > 0 && !problems)) return B200_ERR_INVALID;
    using b200::match::DepthLmDev;
    // validation on the host: the problems that fail it are not launched
    std::vector<int> nv(n_problems, 0);
    int first_bad = B200_OK;
    for (int p = 0; p < n_problems; ++p) {
        b200_depth_landmarks_problem_t& P = problems[p];
        P.n_created = 0;
        int st = B200_OK;
        if ((P.mode != B200_DEPTH_LM_KEYFRAME && P.mode != B200_DEPTH_LM_INITIAL) || P.n_keypoints < 0 || P.num_levels < 1 || !P.scale_factors
            || (P.n_keypoints > 0 && (!P.x || !P.y || !P.octave || !P.depth || !P.created_idx || !P.pos_w || !P.mean_normal || !P.min_valid_dist
                                      || !P.max_valid_dist))) {
            b200::set_error("b200_depth_landmarks: problem %d: bad mode, count or pointer", p);
            st = B200_ERR_INVALID;
        }
        for (int i = 0; st == B200_OK && i < P.n_keypoints; ++i) {
            if (!(0.f < P.depth[i])) continue;
            ++nv[p];
            if (P.model == 1) {
                b200::set_error("b200_depth_landmarks: problem %d: equirectangular camera with a valid depth (data/common.cc:236-238 throws)", p);
                st = B200_ERR_INVALID;
            } else if (P.octave[i] < 0 || P.octave[i] >= P.num_levels) {
                b200::set_error("b200_depth_landmarks: problem %d: keypoint %d has octave %d, the table has %d levels", p, i, P.octave[i], P.num_levels);
                st = B200_ERR_INVALID;
            }
        }
        if (st == B200_OK && P.mode == B200_DEPTH_LM_KEYFRAME && nv[p] > B200_DEPTH_LM_MAX_SORT) {
            b200::set_error("b200_depth_landmarks: problem %d has %d keypoints with a valid depth, at most %d can be sorted", p, nv[p],
                            B200_DEPTH_LM_MAX_SORT);
            st = B200_ERR_CAPACITY;
        }
        P.status = st;
        if (st != B200_OK && first_bad == B200_OK) first_bad = st;
    }
    // one pinned staging block: the problem table, then per problem its inputs (x, y, depth, octave, has_landmark, scale factors) and
    // its outputs (n_created, idx, pos_w, mean_normal, min / max valid distance)
    struct Lay { size_t x, y, depth, oct, has_lm, sf, n_created, idx, pos, nrm, lo, hi; };
    std::vector<Lay> lay(n_problems);
    auto staged = [&](int p) { return problems[p].status == B200_OK ? (size_t)problems[p].n_keypoints : 0; };
    b200::Layout a;
    a.take<DepthLmDev>(n_problems);  // at offset 0
    for (int p = 0; p < n_problems; ++p) {
        const size_t n = staged(p), lv = problems[p].status == B200_OK ? (size_t)problems[p].num_levels : 0;
        Lay& L = lay[p];
        L.x = a.take(4 * n);
        L.y = a.take(4 * n);
        L.depth = a.take(4 * n);
        L.oct = a.take(4 * n);
        L.has_lm = a.take(n);
        L.sf = a.take(4 * lv);
    }
    const size_t in_bytes = a.end;
    for (int p = 0; p < n_problems; ++p) {
        const size_t n = staged(p);
        Lay& L = lay[p];
        L.n_created = a.take(4);
        L.idx = a.take(4 * n);
        L.pos = a.take(24 * n);
        L.nrm = a.take(24 * n);
        L.lo = a.take(4 * n);
        L.hi = a.take(4 * n);
    }
    const size_t out_end = a.end;
    auto& m = h->m;
    B200_CUDA(cudaSetDevice(m.device));
    cudaStream_t st = m.stream;
    int rc;
    if ((rc = m.arena.reserve(out_end, out_end, st))) return rc;
    b200::StagingArena& A = m.arena;
    DepthLmDev* dev = A.host<DepthLmDev>(0);
    int npow_max = 1;
    for (int p = 0; p < n_problems; ++p) {
        const b200_depth_landmarks_problem_t& P = problems[p];
        DepthLmDev& D = dev[p];
        std::memset(&D, 0, sizeof(D));
        if (P.status != B200_OK) continue;  // n_created == nullptr: the kernel skips it
        const Lay& L = lay[p];
        const size_t n = (size_t)P.n_keypoints;
        D.mode = P.mode;
        D.n = P.n_keypoints;
        D.n_valid = nv[p];
        D.npow = 1;
        if (P.mode == B200_DEPTH_LM_KEYFRAME)
            while (D.npow < nv[p]) D.npow <<= 1;
        npow_max = std::max(npow_max, D.npow);
        for (int r = 0; r < 3; ++r) {
            for (int c = 0; c < 3; ++c) D.rwc[3 * r + c] = P.pose_wc[4 * r + c];
            D.twc[r] = P.pose_wc[4 * r + 3];
        }
        D.fx_inv = P.fx_inv; D.fy_inv = P.fy_inv; D.cx = P.cx; D.cy = P.cy; D.depth_thr = P.depth_thr;
        D.inv_last = P.inv_scale_factor_last;
        if (n) {
            A.put(L.x, P.x, 4 * n);          D.x = A.dev<const float>(L.x);
            A.put(L.y, P.y, 4 * n);          D.y = A.dev<const float>(L.y);
            A.put(L.depth, P.depth, 4 * n);  D.depth = A.dev<const float>(L.depth);
            A.put(L.oct, P.octave, 4 * n);   D.octave = A.dev<const int>(L.oct);
            if (P.has_landmark && P.mode == B200_DEPTH_LM_KEYFRAME) {
                A.put(L.has_lm, P.has_landmark, n);
                D.has_lm = A.dev(L.has_lm);
            }
        }
        A.put(L.sf, P.scale_factors, 4 * (size_t)P.num_levels);
        D.sf = A.dev<const float>(L.sf);
        D.n_created = A.dev<int>(L.n_created);
        D.out_idx = A.dev<int>(L.idx);
        D.pos_w = A.dev<double>(L.pos);
        D.mean_normal = A.dev<double>(L.nrm);
        D.min_valid = A.dev<float>(L.lo);
        D.max_valid = A.dev<float>(L.hi);
    }
    if (n_problems == 0) return B200_OK;
    B200_CUDA(A.upload(in_bytes, st));
    B200_CUDA(cudaMemsetAsync(A.dev(in_bytes), 0, out_end - in_bytes, st));
    const size_t smem = sizeof(unsigned long long) * (size_t)npow_max;
    B200_CUDA(cudaFuncSetAttribute(b200::match::depth_landmarks_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    b200::match::depth_landmarks_kernel<<<n_problems, b200::match::kDepthLmThreads, smem, st>>>(A.dev<const DepthLmDev>(0));
    B200_CUDA(cudaGetLastError());
    B200_CUDA(A.download(in_bytes, out_end, st));
    B200_CUDA(cudaStreamSynchronize(st));
    for (int p = 0; p < n_problems; ++p) {
        b200_depth_landmarks_problem_t& P = problems[p];
        if (P.status != B200_OK) continue;
        const Lay& L = lay[p];
        const int k = *A.host<const int>(L.n_created);
        P.n_created = k;
        const size_t K = (size_t)k;
        std::memcpy(P.created_idx, A.host(L.idx), 4 * K);
        std::memcpy(P.pos_w, A.host(L.pos), 24 * K);
        std::memcpy(P.mean_normal, A.host(L.nrm), 24 * K);
        std::memcpy(P.min_valid_dist, A.host(L.lo), 4 * K);
        std::memcpy(P.max_valid_dist, A.host(L.hi), 4 * K);
    }
    return first_bad;
}

namespace {

// b200_remove_redundant_keyframes' input check: ranges, then per rank that the landmarks its keypoints list and the landmarks with an
// observation by it are the same set, each listed and observed exactly once.  Returns B200_OK or B200_ERR_INVALID with the error set.
int check_cull_problem(int p, const b200_cull_problem_t& P) {
    auto bad = [p](const char* what) {
        b200::set_error("b200_remove_redundant_keyframes: problem %d: %s", p, what);
        return B200_ERR_INVALID;
    };
    if (P.n_covisibilities < 0 || P.n_landmarks < 0) return bad("negative count");
    if ((P.n_covisibilities > 0 && !P.covisibilities) || (P.n_landmarks > 0 && !P.obs_offsets)) return bad("null covisibilities or obs_offsets");
    const int L = P.n_landmarks;
    if (L > 0 && P.obs_offsets[0] != 0) return bad("obs_offsets[0] is not 0");
    for (int l = 0; l < L; ++l)
        if (P.obs_offsets[l + 1] < P.obs_offsets[l]) return bad("obs_offsets descend");
    const int total = L > 0 ? P.obs_offsets[L] : 0;
    if (total > 0 && (!P.obs_rank || !P.obs_octave || !P.obs_weight)) return bad("null observation table");
    std::vector<int> rank_start((size_t)P.n_covisibilities + 1, 0);
    for (int j = 0; j < total; ++j) {
        if (P.obs_rank[j] < -1 || P.obs_rank[j] >= P.n_covisibilities) return bad("obs_rank out of range");
        if (P.obs_weight[j] != 1 && P.obs_weight[j] != 2) return bad("obs_weight is not 1 or 2");
        if (P.obs_rank[j] >= 0) ++rank_start[P.obs_rank[j] + 1];
    }
    for (int r = 0; r < P.n_covisibilities; ++r) rank_start[r + 1] += rank_start[r];
    std::vector<int> by_rank((size_t)rank_start[P.n_covisibilities]), fill(rank_start.begin(), rank_start.end() - 1);
    for (int l = 0; l < L; ++l)
        for (int j = P.obs_offsets[l]; j < P.obs_offsets[l + 1]; ++j)
            if (P.obs_rank[j] >= 0) by_rank[fill[P.obs_rank[j]]++] = l;
    std::vector<int> mark((size_t)L, -1);
    for (int r = 0; r < P.n_covisibilities; ++r) {
        const b200_cull_keyframe_t& K = P.covisibilities[r];
        if (K.n_keypoints < 0 || (K.n_keypoints > 0 && !K.kp_landmark)) return bad("bad keypoint count or null kp_landmark");
        int listed = 0;
        for (int i = 0; i < K.n_keypoints; ++i) {
            const int l = K.kp_landmark[i];
            if (l < -1 || l >= L) return bad("kp_landmark out of range");
            if (l < 0) continue;
            if (mark[l] == r) return bad("a landmark is listed by two keypoints of one covisibility");
            mark[l] = r;
            ++listed;
        }
        if (listed != rank_start[r + 1] - rank_start[r]) return bad("a covisibility's keypoints and its observations disagree");
        for (int k = rank_start[r]; k < rank_start[r + 1]; ++k) {
            if (mark[by_rank[k]] != r) return bad("a covisibility's keypoints and its observations disagree");
            mark[by_rank[k]] = -1;  // a second observation by r of the same landmark fails here
        }
    }
    return B200_OK;
}

}  // namespace

int b200_remove_redundant_keyframes(b200_matcher_t h, int n_problems, b200_cull_problem_t* problems) {
    B200_RANGE("b200:match:remove_redundant_keyframes");
    if (!h || n_problems < 0 || (n_problems > 0 && !problems)) return B200_ERR_INVALID;
    for (int p = 0; p < n_problems; ++p)
        if (int rc = check_cull_problem(p, problems[p])) return rc;
    if (n_problems == 0) return B200_OK;
    using b200::match::CullDev;
    using b200::match::CullKfDev;
    // one staging block: the problem table, then per problem its covisibility table, observation table and keypoint arrays; the
    // outputs (n_removed, then n_valid / n_redundant / skipped / removed per rank); the device-only live landmark state
    struct Lay { size_t kf, off, rank, octave, weight, out, live_w, live_c, erased; std::vector<size_t> kp_lm, depth; };
    std::vector<Lay> lay(n_problems);
    b200::Layout a;
    a.take<CullDev>(n_problems);  // at offset 0
    for (int p = 0; p < n_problems; ++p) {
        const b200_cull_problem_t& P = problems[p];
        const size_t L = (size_t)P.n_landmarks, total = L ? (size_t)P.obs_offsets[L] : 0;
        Lay& Y = lay[p];
        Y.kf = a.take<CullKfDev>(P.n_covisibilities);
        Y.off = a.take<int>(L + 1);
        Y.rank = a.take<int>(total);
        Y.octave = a.take<int>(total);
        Y.weight = a.take(total);
        for (int r = 0; r < P.n_covisibilities; ++r) {
            const b200_cull_keyframe_t& K = P.covisibilities[r];
            Y.kp_lm.push_back(a.take<int>(K.n_keypoints));
            Y.depth.push_back(K.depth ? a.take<float>(K.n_keypoints) : 0);
        }
    }
    const size_t in_bytes = a.end;
    for (int p = 0; p < n_problems; ++p) lay[p].out = a.take<int>(1 + 4 * (size_t)problems[p].n_covisibilities);
    const size_t out_end = a.end;
    for (int p = 0; p < n_problems; ++p) {
        const size_t L = (size_t)problems[p].n_landmarks;
        lay[p].live_w = a.take<int>(L);
        lay[p].live_c = a.take<int>(L);
        lay[p].erased = a.take(L ? (size_t)problems[p].obs_offsets[L] : 0);
    }
    auto& m = h->m;
    B200_CUDA(cudaSetDevice(m.device));
    cudaStream_t st = m.stream;
    int rc;
    if ((rc = m.arena.reserve(a.end, out_end, st))) return rc;
    b200::StagingArena& A = m.arena;
    CullDev* dev = A.host<CullDev>(0);
    for (int p = 0; p < n_problems; ++p) {
        const b200_cull_problem_t& P = problems[p];
        const Lay& Y = lay[p];
        const size_t L = (size_t)P.n_landmarks, total = L ? (size_t)P.obs_offsets[L] : 0;
        CullDev& D = dev[p];
        std::memset(&D, 0, sizeof(D));
        D.cur_id = P.cur_id;
        D.n_cov = P.n_covisibilities;
        D.n_lm = P.n_landmarks;
        D.thr = P.redundant_obs_ratio_thr;
        D.kf = A.dev<const CullKfDev>(Y.kf);
        if (L) A.put(Y.off, P.obs_offsets, 4 * (L + 1));
        else *A.host<int>(Y.off) = 0;
        A.put(Y.rank, P.obs_rank, 4 * total);
        A.put(Y.octave, P.obs_octave, 4 * total);
        A.put(Y.weight, P.obs_weight, total);
        D.off = A.dev<const int>(Y.off);
        D.rank = A.dev<const int>(Y.rank);
        D.octave = A.dev<const int>(Y.octave);
        D.weight = A.dev<const unsigned char>(Y.weight);
        D.live_weight = A.dev<int>(Y.live_w);
        D.live_count = A.dev<int>(Y.live_c);
        D.erased = A.dev<unsigned char>(Y.erased);
        D.n_removed = A.dev<int>(Y.out);
        CullKfDev* kf = A.host<CullKfDev>(Y.kf);
        for (int r = 0; r < P.n_covisibilities; ++r) {
            const b200_cull_keyframe_t& K = P.covisibilities[r];
            CullKfDev& E = kf[r];
            std::memset(&E, 0, sizeof(E));
            E.id = K.id;
            E.is_root = K.is_root != 0;
            E.n = K.n_keypoints;
            E.depth_thr = K.depth_thr;
            A.put(Y.kp_lm[r], K.kp_landmark, 4 * (size_t)K.n_keypoints);
            E.kp_lm = A.dev<const int>(Y.kp_lm[r]);
            if (K.depth) {
                A.put(Y.depth[r], K.depth, 4 * (size_t)K.n_keypoints);
                E.depth = A.dev<const float>(Y.depth[r]);
            }
            E.out = A.dev<int>(Y.out) + 1 + 4 * r;
        }
    }
    B200_CUDA(A.upload(in_bytes, st));
    B200_CUDA(cudaMemsetAsync(A.dev(in_bytes), 0, out_end - in_bytes, st));
    b200::match::cull_keyframes_kernel<<<n_problems, b200::match::kCullThreads, 0, st>>>(A.dev<const CullDev>(0));
    B200_CUDA(cudaGetLastError());
    B200_CUDA(A.download(in_bytes, out_end, st));
    B200_CUDA(cudaStreamSynchronize(st));
    for (int p = 0; p < n_problems; ++p) {
        b200_cull_problem_t& P = problems[p];
        const int* o = A.host<const int>(lay[p].out);
        P.n_removed = o[0];
        for (int r = 0; r < P.n_covisibilities; ++r) {
            b200_cull_keyframe_t& K = P.covisibilities[r];
            K.n_valid = o[1 + 4 * r];
            K.n_redundant = o[2 + 4 * r];
            K.skipped = o[3 + 4 * r];
            K.removed = o[4 + 4 * r];
        }
        P.status = B200_OK;
    }
    return B200_OK;
}

int b200_match_cross_check(const int32_t* idx2_in_1, int n1, const int32_t* idx1_in_2, int n2, int32_t* mutual_out, int32_t* n_mutual) {
    if (n1 < 0 || n2 < 0 || (n1 > 0 && (!idx2_in_1 || !mutual_out)) || (n2 > 0 && !idx1_in_2)) return B200_ERR_INVALID;
    int n = 0;
    for (int i = 0; i < n1; ++i) {
        const int j = idx2_in_1[i];
        const bool keep = 0 <= j && j < n2 && idx1_in_2[j] == i;
        mutual_out[i] = keep ? j : -1;
        n += keep;
    }
    if (n_mutual) *n_mutual = n;
    return B200_OK;
}

int b200_hamming_matrix(b200_matcher_t h, const uint8_t* desc1, int n1, const uint8_t* desc2, int n2, uint16_t* dist) {
    if (!h || n1 < 0 || n2 < 0) return B200_ERR_INVALID;
    if (n1 == 0 || n2 == 0) return B200_OK;
    if (!desc1 || !desc2 || !dist) return B200_ERR_INVALID;
    auto& m = h->m;
    B200_CUDA(cudaSetDevice(m.device));
    b200::Layout L;
    const size_t o_d1 = L.take((size_t)32 * n1), o_d2 = L.take((size_t)32 * n2), o_out = L.take<uint16_t>((size_t)n1 * n2);
    int rc = m.arena.reserve(L.end, 0, m.stream);
    if (rc) return rc;
    unsigned char* s = m.arena.d;
    B200_CUDA(cudaMemcpyAsync(s + o_d1, desc1, (size_t)32 * n1, cudaMemcpyHostToDevice, m.stream));
    B200_CUDA(cudaMemcpyAsync(s + o_d2, desc2, (size_t)32 * n2, cudaMemcpyHostToDevice, m.stream));
    b200::match::hamming_matrix_kernel<<<dim3(b200::ceil_div(n2, 64), b200::ceil_div(n1, 256)), 256, 0, m.stream>>>(
        (const uint4*)(s + o_d1), n1, (const uint4*)(s + o_d2), n2, (unsigned short*)(s + o_out));
    B200_CUDA(cudaGetLastError());
    B200_CUDA(cudaMemcpyAsync(dist, s + o_out, sizeof(uint16_t) * (size_t)n1 * n2, cudaMemcpyDeviceToHost, m.stream));
    B200_CUDA(cudaStreamSynchronize(m.stream));
    return B200_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------
// New landmarks of the mapping module (mapping_module::create_new_landmarks, src/stella_vslam/mapping_module.cc, and
// module::two_view_triangulator): the triangulation device function lives in triangulate.cuh.
//   b200_triangulate_pairs    : one thread per match over every problem of the call (flattened offsets)
//   b200_create_new_landmarks : pairs_candidates_kernel over every (keyframe, neighbour) problem, then per neighbour rank the
//                               resolve (guided_resolve_kernel, mode 6) and landmark_claim_kernel, which triangulates that rank's
//                               matches, appends the landmarks in idx_1 order and closes the rows it created a landmark on to the
//                               later ranks (list_len = 0: match_for_triangulation skips a keypoint with a landmark, robust.cc:44-48)
// ---------------------------------------------------------------------------------------------------------------
namespace b200 {
namespace mapping {

using match::PairsDev;
using tri::TriKfDev;

struct TriProblemDev {
    int k1, k2;  // rows of the keyframe table
    float cos_thr, ratio_factor;
    int begin;   // first match of the problem in the flattened arrays
};

__global__ void __launch_bounds__(256) triangulate_pairs_kernel(const TriKfDev* __restrict__ kfs, const TriProblemDev* __restrict__ ps, int n_problems,
                                                                int total, const int2* __restrict__ matches, double* __restrict__ pos_w,
                                                                unsigned char* __restrict__ ok, int* __restrict__ unconverged) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= total) return;
    int lo = 0, hi = n_problems - 1;  // last problem that starts at or before t
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (ps[mid].begin <= t) lo = mid;
        else hi = mid - 1;
    }
    const TriProblemDev& P = ps[lo];
    const int2 m = matches[t];
    double p[3];
    const int r = tri::two_view_triangulate(kfs[P.k1], kfs[P.k2], m.x, m.y, P.cos_thr, P.ratio_factor, p);
    if (r < 0) atomicAdd(unconverged, 1);
    pos_w[3 * (size_t)t] = p[0];
    pos_w[3 * (size_t)t + 1] = p[1];
    pos_w[3 * (size_t)t + 2] = p[2];
    ok[t] = r == 1;
}

struct ChainKfDev {
    int cur;       // row of the current keyframe in the keyframe table
    int n_nb;      // neighbours (ranks)
    int nb_begin;  // row of its rank-0 neighbour in the keyframe table and in nb_consts (the ranks follow)
    int* n_created_rank;  // [n_nb]
    int* n_created;       // [1], running count
    int* created_rank;
    int2* created_idx;
    double* created_pos;
};

constexpr int kClaimThreads = 256;

__global__ void __launch_bounds__(kClaimThreads) landmark_claim_kernel(const TriKfDev* __restrict__ kfs, const float2* __restrict__ nb_consts, const ChainKfDev* __restrict__ ks,
                                                                       const PairsDev* __restrict__ pairs, int n_kf, int rank,
                                                                       int* __restrict__ unconverged) {
    __shared__ int warp_total[kClaimThreads / 32];
    const ChainKfDev K = ks[blockIdx.x];
    if (rank >= K.n_nb) return;
    const PairsDev& g = pairs[(size_t)rank * n_kf + blockIdx.x];
    const TriKfDev& k1 = kfs[K.cur];
    const TriKfDev& k2 = kfs[K.nb_begin + rank];
    const float2 c = nb_consts[K.nb_begin + rank];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int base = *K.n_created;  // written by this keyframe's block of the previous rank (stream order)
    int made = 0;
    for (int c0 = 0; c0 < g.n_queries; c0 += kClaimThreads) {
        const int i = c0 + threadIdx.x;
        const int j = i < g.n_queries ? g.match_out[i] : -1;
        double p[3];
        bool ok = false;
        if (j >= 0) {
            const int r = tri::two_view_triangulate(k1, k2, i, j, c.x, c.y, p);
            if (r < 0) atomicAdd(unconverged, 1);
            ok = r == 1;
        }
        // ordered compaction: rows in ascending idx_1 (the order of matched_idx_pairs, robust.cc:135-143)
        const unsigned bal = __ballot_sync(0xFFFFFFFFu, ok);
        if (lane == 0) warp_total[warp] = __popc(bal);
        __syncthreads();
        int off = 0, chunk = 0;
#pragma unroll
        for (int w = 0; w < kClaimThreads / 32; ++w) {
            off += w < warp ? warp_total[w] : 0;
            chunk += warp_total[w];
        }
        if (ok) {
            const int at = base + off + __popc(bal & ((1u << lane) - 1u));
            K.created_rank[at] = rank;
            K.created_idx[at] = make_int2(i, j);
            K.created_pos[3 * (size_t)at] = p[0];
            K.created_pos[3 * (size_t)at + 1] = p[1];
            K.created_pos[3 * (size_t)at + 2] = p[2];
            for (int r2 = rank + 1; r2 < K.n_nb; ++r2) pairs[(size_t)r2 * n_kf + blockIdx.x].list_len[i] = 0;
        }
        base += chunk;
        made += chunk;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        *K.n_created = base;
        K.n_created_rank[rank] = made;
    }
}

struct KfLay {
    size_t x, y, oct, xr, dep, b, sf, ls;
};

bool kf_valid(const b200_tri_keyframe_t* K) {
    if (!K || K->n_keypoints < 0 || (K->model != 0 && K->model != 1) || K->num_levels < 1 || K->num_levels > 64 || !K->scale_factors
        || !K->level_sigma_sq)
        return false;
    return K->n_keypoints == 0 || (K->x && K->y && K->octave && K->bearings);
}

// octave of keypoint i in range, and no stereo keypoint on an equirectangular camera (data/common.cc:240-242 throws there)
bool kp_valid(const b200_tri_keyframe_t* K, int i) {
    return i >= 0 && i < K->n_keypoints && K->octave[i] >= 0 && K->octave[i] < K->num_levels
           && !(K->model == 1 && K->x_right && K->x_right[i] >= 0.0f);
}

KfLay layout_kf(Layout& a, const b200_tri_keyframe_t* K) {
    const size_t n = (size_t)K->n_keypoints, nl = (size_t)K->num_levels;
    KfLay L;
    L.x = a.take(4 * n);
    L.y = a.take(4 * n);
    L.oct = a.take(4 * n);
    L.xr = a.take(4 * n);
    L.dep = a.take(4 * n);
    L.b = a.take(24 * n);
    L.sf = a.take(4 * nl);
    L.ls = a.take(4 * nl);
    return L;
}

// Stages the keyframe's arrays at L and returns its device view.
TriKfDev make_kf(const b200_tri_keyframe_t* K, const KfLay& L, StagingArena& A) {
    const size_t n = (size_t)K->n_keypoints, nl = (size_t)K->num_levels;
    A.put(L.x, K->x, 4 * n);
    A.put(L.y, K->y, 4 * n);
    A.put(L.oct, K->octave, 4 * n);
    A.put(L.xr, K->x_right, 4 * n);
    A.put(L.dep, K->depth, 4 * n);
    A.put(L.b, K->bearings, 24 * n);
    A.put(L.sf, K->scale_factors, 4 * nl);
    A.put(L.ls, K->level_sigma_sq, 4 * nl);
    const unsigned char* db = A.d;
    TriKfDev d{};
    std::memcpy(d.pose_cw, K->pose_cw, sizeof(d.pose_cw));
    std::memcpy(d.pose_wc, K->pose_wc, sizeof(d.pose_wc));
    d.model = K->model;
    d.fx = K->fx;
    d.fy = K->fy;
    d.cx = K->cx;
    d.cy = K->cy;
    d.fx_inv = K->fx_inv;
    d.fy_inv = K->fy_inv;
    d.fxb = K->focal_x_baseline;
    d.true_baseline = K->true_baseline;
    d.cols = K->cols;
    d.rows = K->rows;
    d.x = (const float*)(db + L.x);
    d.y = (const float*)(db + L.y);
    d.octave = (const int*)(db + L.oct);
    d.x_right = K->x_right ? (const float*)(db + L.xr) : nullptr;
    d.depth = K->depth ? (const float*)(db + L.dep) : nullptr;
    d.bearings = (const double*)(db + L.b);
    d.scale_factors = (const float*)(db + L.sf);
    d.level_sigma_sq = (const float*)(db + L.ls);
    return d;
}

// the triangulator's constructor (two_view_triangulator.cc:15-16): ratio_factor_ and cos_rays_parallax_thr_ are floats
float2 tri_constants(const b200_tri_keyframe_t* k1, const b200_tri_keyframe_t* k2, float rays_parallax_deg_thr) {
    const float cos_thr = (float)std::cos(rays_parallax_deg_thr * M_PI / 180.0);
    const float ratio_factor = 2.0f * std::max(k1->scale_factor, k2->scale_factor);
    return make_float2(cos_thr, ratio_factor);
}

}  // namespace mapping
}  // namespace b200

int b200_triangulate_pairs(b200_matcher_t h, int n_problems, b200_triangulate_problem_t* problems) {
    B200_RANGE("b200:mapping:triangulate");
    using namespace b200::mapping;
    if (!h || n_problems < 0) return B200_ERR_INVALID;
    if (n_problems == 0) return B200_OK;
    if (!problems) return B200_ERR_INVALID;
    auto& m = h->m;
    B200_CUDA(cudaSetDevice(m.device));
    // keyframe table: each distinct keyframe view goes up once
    std::vector<const b200_tri_keyframe_t*> kf_list;
    auto kf_row = [&](const b200_tri_keyframe_t* K) {
        for (size_t r = 0; r < kf_list.size(); ++r)
            if (kf_list[r] == K) return (int)r;
        kf_list.push_back(K);
        return (int)kf_list.size() - 1;
    };
    std::vector<TriProblemDev> tp(n_problems);
    int total = 0;
    for (int p = 0; p < n_problems; ++p) {
        const b200_triangulate_problem_t& P = problems[p];
        if (!kf_valid(P.keyfrm_1) || !kf_valid(P.keyfrm_2) || P.n_matches < 0 || (P.n_matches > 0 && (!P.matches || !P.pos_w || !P.ok))) {
            b200::set_error("b200_triangulate_pairs: bad keyframe view, size or null buffer in problem %d", p);
            return B200_ERR_INVALID;
        }
        for (int k = 0; k < P.n_matches; ++k)
            if (!kp_valid(P.keyfrm_1, P.matches[2 * k]) || !kp_valid(P.keyfrm_2, P.matches[2 * k + 1])) {
                b200::set_error("b200_triangulate_pairs: problem %d match %d: index or octave out of range, or a stereo keypoint on an "
                                "equirectangular camera", p, k);
                return B200_ERR_INVALID;
            }
        if (total > INT_MAX - P.n_matches) return B200_ERR_INVALID;
        const float2 c = tri_constants(P.keyfrm_1, P.keyfrm_2, P.rays_parallax_deg_thr);
        tp[p] = TriProblemDev{kf_row(P.keyfrm_1), kf_row(P.keyfrm_2), c.x, c.y, total};
        total += P.n_matches;
    }
    b200::Layout a;
    const size_t o_kfs = a.take<TriKfDev>(kf_list.size());
    const size_t o_ps = a.take<TriProblemDev>(n_problems);
    std::vector<KfLay> kl;
    for (const b200_tri_keyframe_t* K : kf_list) kl.push_back(layout_kf(a, K));
    // every problem's (idx_1, idx_2) rows, consecutive in problem order
    const size_t o_matches = a.take(8 * (size_t)total);
    const size_t in_bytes = a.end, out_begin = a.end;
    const size_t o_pos = a.take(24 * (size_t)total);
    const size_t o_ok = a.take((size_t)total);
    const size_t o_unconv = a.take(4);
    const size_t out_end = a.end;
    cudaStream_t st = m.stream;
    int rc;
    if ((rc = m.arena.reserve(a.end, a.end, st))) return rc;
    b200::StagingArena& A = m.arena;
    unsigned char *hb = A.h, *db = A.d;
    for (int p = 0; p < n_problems; ++p)
        A.put(o_matches + 8 * (size_t)tp[p].begin, problems[p].matches, 8 * (size_t)problems[p].n_matches);
    TriKfDev* hk = A.host<TriKfDev>(o_kfs);
    for (size_t r = 0; r < kf_list.size(); ++r) hk[r] = make_kf(kf_list[r], kl[r], A);
    A.put(o_ps, tp.data(), sizeof(TriProblemDev) * (size_t)n_problems);
    B200_CUDA(A.upload(in_bytes, st));
    B200_CUDA(cudaMemsetAsync(db + o_unconv, 0, 4, st));
    if (total > 0) {
        triangulate_pairs_kernel<<<b200::ceil_div(total, 256), 256, 0, st>>>(
            (const TriKfDev*)(db + o_kfs), (const TriProblemDev*)(db + o_ps), n_problems, total, (const int2*)(db + o_matches),
            (double*)(db + o_pos), db + o_ok, (int*)(db + o_unconv));
        B200_CUDA(cudaGetLastError());
    }
    B200_CUDA(A.download(out_begin, out_end, st));
    B200_CUDA(cudaStreamSynchronize(st));
    const int unconverged = *reinterpret_cast<const int*>(hb + o_unconv);
    if (unconverged > 0) {
        b200::set_error("b200_triangulate_pairs: the 4x4 Jacobi SVD did not converge within %d sweeps for %d matches", b200::tri::kMaxSweeps,
                        unconverged);
        return B200_ERR_INVALID;
    }
    for (int p = 0; p < n_problems; ++p) {
        b200_triangulate_problem_t& P = problems[p];
        const size_t b = (size_t)tp[p].begin, n = (size_t)P.n_matches;
        int n_ok = 0;
        if (n) {
            std::memcpy(P.pos_w, hb + o_pos + 24 * b, 24 * n);
            std::memcpy(P.ok, hb + o_ok + b, n);
            for (size_t k = 0; k < n; ++k) n_ok += P.ok[k];
        }
        P.n_ok = n_ok;
    }
    return B200_OK;
}

int b200_create_new_landmarks(b200_matcher_t h, int n_keyframes, b200_new_landmarks_problem_t* problems, float lowe_ratio, float residual_rad_thr,
                              float rays_parallax_deg_thr, int max_candidates) {
    B200_RANGE("b200:mapping:new_landmarks");
    using namespace b200::mapping;
    if (!h || n_keyframes < 0 || max_candidates < 0) return B200_ERR_INVALID;
    if (n_keyframes == 0) return B200_OK;
    if (!problems) return B200_ERR_INVALID;
    auto& m = h->m;
    B200_CUDA(cudaSetDevice(m.device));
    const int cap = max_candidates ? max_candidates : 64;
    const int n_kf = n_keyframes;
    int n_ranks = 0, max_n1 = 0, max_n2 = 0;
    for (int k = 0; k < n_kf; ++k) {
        const b200_new_landmarks_problem_t& P = problems[k];
        const b200_tri_keyframe_t* C = P.keyfrm;
        bool bad = !kf_valid(C) || P.n_neighbours < 0 || (P.n_neighbours > 0 && !P.neighbours)
                   || (C->n_keypoints > 0 && (!P.desc || !P.created_rank || !P.created_idx || !P.created_pos_w));
        for (int i = 0; !bad && i < C->n_keypoints; ++i) bad = !kp_valid(C, i);
        for (int r = 0; !bad && r < P.n_neighbours; ++r) {
            const b200_new_landmarks_neighbour_t& N = P.neighbours[r];
            bad = !kf_valid(N.keyfrm) || (N.keyfrm->n_keypoints > 0 && !N.desc) || ((P.node == nullptr) != (N.node == nullptr));
            for (int i = 0; !bad && i < N.keyfrm->n_keypoints; ++i) bad = !kp_valid(N.keyfrm, i);
            if (!bad) max_n2 = std::max(max_n2, N.keyfrm->n_keypoints);
        }
        if (bad) {
            b200::set_error("b200_create_new_landmarks: keyframe %d: bad keyframe view, size, null buffer, octave out of range or a stereo "
                            "keypoint on an equirectangular camera", k);
            return B200_ERR_INVALID;
        }
        n_ranks = std::max(n_ranks, P.n_neighbours);
        max_n1 = std::max(max_n1, C->n_keypoints);
    }
    if (n_ranks == 0) {
        for (int k = 0; k < n_kf; ++k) problems[k].n_created = 0;
        return B200_OK;
    }
    const size_t rs_bytes = (size_t)std::max(max_n2, 1) * 6 + 16;
    if (rs_bytes > 200 * 1024) {
        b200::set_error("b200_create_new_landmarks: %d keypoints per neighbour exceed the on-chip occupancy table", max_n2);
        return B200_ERR_CAPACITY;
    }
    // host-derived per-keypoint inputs of the matcher: scale_factors_[octave] of the rows, stereo flags of both sides
    std::vector<std::vector<float>> scale1(n_kf);
    std::vector<std::vector<unsigned char>> stereo_cur(n_kf);
    std::vector<std::vector<std::vector<unsigned char>>> stereo_nb(n_kf);
    auto stereo_of = [](const b200_tri_keyframe_t* K, std::vector<unsigned char>& out) {
        if (!K->x_right) return;
        out.resize(K->n_keypoints);
        for (int i = 0; i < K->n_keypoints; ++i) out[i] = K->x_right[i] >= 0.0f;
    };
    b200::Layout s;
    const size_t P_total = (size_t)n_ranks * n_kf;
    const size_t o_pairs = s.take<PairsDev>(P_total);
    const size_t o_chain = s.take<ChainKfDev>(n_kf);
    int n_views = 0;
    for (int k = 0; k < n_kf; ++k) n_views += 1 + problems[k].n_neighbours;
    const size_t o_kfs = s.take<TriKfDev>(n_views);
    const size_t o_consts = s.take(8 * (size_t)n_views);
    struct CurLay {
        KfLay kf;
        size_t desc, valid, node, scale, stereo;
    };
    struct NbLay {
        KfLay kf;
        size_t desc, valid, node, stereo;
    };
    std::vector<CurLay> cl(n_kf);
    std::vector<std::vector<NbLay>> nl(n_kf);
    for (int k = 0; k < n_kf; ++k) {
        const b200_new_landmarks_problem_t& P = problems[k];
        const b200_tri_keyframe_t* C = P.keyfrm;
        const size_t n1 = (size_t)C->n_keypoints;
        scale1[k].resize(n1);
        for (size_t i = 0; i < n1; ++i) scale1[k][i] = C->scale_factors[C->octave[i]];
        stereo_of(C, stereo_cur[k]);
        CurLay& L = cl[k];
        L.kf = layout_kf(s, C);
        L.desc = s.take(32 * n1);
        L.valid = s.take(n1);
        L.node = s.take(4 * n1);
        L.scale = s.take(4 * n1);
        L.stereo = s.take(n1);
        stereo_nb[k].resize(P.n_neighbours);
        nl[k].resize(P.n_neighbours);
        for (int r = 0; r < P.n_neighbours; ++r) {
            const b200_new_landmarks_neighbour_t& N = P.neighbours[r];
            const size_t n2 = (size_t)N.keyfrm->n_keypoints;
            stereo_of(N.keyfrm, stereo_nb[k][r]);
            NbLay& M = nl[k][r];
            M.kf = layout_kf(s, N.keyfrm);
            M.desc = s.take(32 * n2);
            M.valid = s.take(n2);
            M.node = s.take(4 * n2);
            M.stereo = s.take(n2);
        }
    }
    const size_t in_bytes = s.end, out_begin = s.end;
    // outputs (one download): per problem match_out + n_matches, per keyframe the created list and counts, the two flags
    std::vector<size_t> o_mout(P_total), o_nm(P_total);
    for (int r = 0; r < n_ranks; ++r)
        for (int k = 0; k < n_kf; ++k) {
            const size_t q = (size_t)r * n_kf + k;
            o_mout[q] = s.take(4 * (size_t)(r < problems[k].n_neighbours ? problems[k].keyfrm->n_keypoints : 0));
            o_nm[q] = s.take(4);
        }
    struct OutLay {
        size_t n_rank, n_created, rank, idx, pos;
    };
    std::vector<OutLay> ol(n_kf);
    for (int k = 0; k < n_kf; ++k) {
        const size_t n1 = (size_t)problems[k].keyfrm->n_keypoints;
        ol[k].n_rank = s.take(4 * (size_t)problems[k].n_neighbours);
        ol[k].n_created = s.take(4);
        ol[k].rank = s.take(4 * n1);
        ol[k].idx = s.take(8 * n1);
        ol[k].pos = s.take(24 * n1);
    }
    const size_t o_overflow = s.take(4), o_unconv = s.take(4);
    const size_t out_end = s.end;
    std::vector<size_t> o_lists(P_total), o_llen(P_total);
    for (int r = 0; r < n_ranks; ++r)
        for (int k = 0; k < n_kf; ++k) {
            const size_t q = (size_t)r * n_kf + k;
            const size_t n1 = r < problems[k].n_neighbours ? (size_t)problems[k].keyfrm->n_keypoints : 0;
            o_lists[q] = s.take(8 * (size_t)cap * n1);
            o_llen[q] = s.take(4 * n1);
        }
    cudaStream_t st = m.stream;
    int rc;
    if ((rc = m.arena.reserve(s.end, out_end, st))) return rc;
    b200::StagingArena& A = m.arena;
    unsigned char *hb = A.h, *db = A.d;
    TriKfDev* hk = A.host<TriKfDev>(o_kfs);
    float2* hc = A.host<float2>(o_consts);
    ChainKfDev* hch = A.host<ChainKfDev>(o_chain);
    PairsDev* hg = A.host<PairsDev>(o_pairs);
    int view = 0;
    for (int k = 0; k < n_kf; ++k) {
        const b200_new_landmarks_problem_t& P = problems[k];
        const b200_tri_keyframe_t* C = P.keyfrm;
        const size_t n1 = (size_t)C->n_keypoints;
        const int cur = view++;
        hk[cur] = make_kf(C, cl[k].kf, A);
        A.put(cl[k].desc, P.desc, 32 * n1);
        A.put(cl[k].valid, P.valid, n1);
        A.put(cl[k].node, P.node, 4 * n1);
        A.put(cl[k].scale, scale1[k].data(), 4 * n1);
        A.put(cl[k].stereo, C->x_right ? stereo_cur[k].data() : nullptr, n1);
        ChainKfDev K{};
        K.cur = cur;
        K.n_nb = P.n_neighbours;
        K.nb_begin = view;
        K.n_created_rank = (int*)(db + ol[k].n_rank);
        K.n_created = (int*)(db + ol[k].n_created);
        K.created_rank = (int*)(db + ol[k].rank);
        K.created_idx = (int2*)(db + ol[k].idx);
        K.created_pos = (double*)(db + ol[k].pos);
        for (int r = 0; r < n_ranks; ++r) {
            const size_t q = (size_t)r * n_kf + k;
            PairsDev g{};
            g.cap = cap;
            g.lists = (uint2*)(db + o_lists[q]);
            g.list_len = (int*)(db + o_llen[q]);
            g.match_out = (int*)(db + o_mout[q]);
            g.n_matches = (int*)(db + o_nm[q]);
            if (r < P.n_neighbours) {
                const b200_new_landmarks_neighbour_t& N = P.neighbours[r];
                const NbLay& M = nl[k][r];
                const size_t n2 = (size_t)N.keyfrm->n_keypoints;
                hk[view] = make_kf(N.keyfrm, M.kf, A);
                A.put(M.desc, N.desc, 32 * n2);
                A.put(M.valid, N.valid, n2);
                A.put(M.node, N.node, 4 * n2);
                A.put(M.stereo, N.keyfrm->x_right ? stereo_nb[k][r].data() : nullptr, n2);
                hc[view] = tri_constants(C, N.keyfrm, rays_parallax_deg_thr);
                ++view;
                g.n_queries = C->n_keypoints;
                g.n_train = N.keyfrm->n_keypoints;
                g.desc1 = (const uint4*)(db + cl[k].desc);
                g.desc2 = (const uint4*)(db + M.desc);
                g.valid1 = P.valid ? db + cl[k].valid : nullptr;
                g.valid2 = N.valid ? db + M.valid : nullptr;
                g.stereo1 = C->x_right ? db + cl[k].stereo : nullptr;
                g.stereo2 = N.keyfrm->x_right ? db + M.stereo : nullptr;
                g.node1 = P.node ? (const int*)(db + cl[k].node) : nullptr;
                g.node2 = N.node ? (const int*)(db + M.node) : nullptr;
                g.bearing1 = hk[cur].bearings;
                g.bearing2 = (const double*)(db + M.kf.b);
                g.scale1 = (const float*)(db + cl[k].scale);
                for (int e = 0; e < 9; ++e) g.E[e] = N.E_12[e];
                for (int e = 0; e < 3; ++e) g.epi[e] = N.epiplane_in_keyfrm_2[e];
                g.valid_epiplane = N.valid_epiplane;
                g.residual_rad_thr = residual_rad_thr;
            }
            hg[q] = g;
        }
        hch[k] = K;
    }
    const PairsDev* dg = A.dev<const PairsDev>(o_pairs);
    B200_CUDA(A.upload(in_bytes, st));
    B200_CUDA(cudaMemsetAsync(db + out_begin, 0, out_end - out_begin, st));
    b200::match::pairs_candidates_kernel<<<dim3(std::max(1, b200::ceil_div(max_n1, b200::match::kPairRows)), (unsigned)P_total),
                                           b200::match::kPairRows, 0, st>>>(dg, B200_PAIRS_TRIANGULATION, (unsigned)b200::match::kThrLow, 0,
                                                                            (int*)(db + o_overflow));
    if (rs_bytes > 48 * 1024)
        B200_CUDA(cudaFuncSetAttribute(b200::match::guided_resolve_kernel<PairsDev>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rs_bytes));
    for (int r = 0; r < n_ranks; ++r) {
        b200::match::guided_resolve_kernel<PairsDev><<<n_kf, 32, rs_bytes, st>>>(dg + (size_t)r * n_kf, 6, (unsigned)b200::match::kThrLow, lowe_ratio);
        landmark_claim_kernel<<<n_kf, kClaimThreads, 0, st>>>((const TriKfDev*)(db + o_kfs), (const float2*)(db + o_consts), (const ChainKfDev*)(db + o_chain), dg, n_kf, r,
                                                              (int*)(db + o_unconv));
    }
    B200_CUDA(cudaGetLastError());
    B200_CUDA(A.download(out_begin, out_end, st));
    B200_CUDA(cudaStreamSynchronize(st));
    const int overflow = *reinterpret_cast<const int*>(hb + o_overflow);
    if (overflow > 0) {
        b200::set_error("b200_create_new_landmarks: a row kept %d gated candidates, max_candidates is %d", overflow, cap);
        return B200_ERR_CAPACITY;
    }
    const int unconverged = *reinterpret_cast<const int*>(hb + o_unconv);
    if (unconverged > 0) {
        b200::set_error("b200_create_new_landmarks: the 4x4 Jacobi SVD did not converge within %d sweeps for %d matches",
                        b200::tri::kMaxSweeps, unconverged);
        return B200_ERR_INVALID;
    }
    for (int k = 0; k < n_kf; ++k) {
        b200_new_landmarks_problem_t& P = problems[k];
        const size_t n1 = (size_t)P.keyfrm->n_keypoints;
        for (int r = 0; r < P.n_neighbours; ++r) {
            b200_new_landmarks_neighbour_t& N = P.neighbours[r];
            const size_t q = (size_t)r * n_kf + k;
            N.n_matches = *reinterpret_cast<const int*>(hb + o_nm[q]);
            N.n_created = reinterpret_cast<const int*>(hb + ol[k].n_rank)[r];
            if (N.match_out && n1) std::memcpy(N.match_out, hb + o_mout[q], 4 * n1);
        }
        const int nc = *reinterpret_cast<const int*>(hb + ol[k].n_created);
        P.n_created = nc;
        if (nc) {
            std::memcpy(P.created_rank, hb + ol[k].rank, 4 * (size_t)nc);
            std::memcpy(P.created_idx, hb + ol[k].idx, 8 * (size_t)nc);
            std::memcpy(P.created_pos_w, hb + ol[k].pos, 24 * (size_t)nc);
        }
    }
    return B200_OK;
}
