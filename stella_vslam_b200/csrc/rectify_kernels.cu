// rectify_kernels.cu -- util::stereo_rectifier: undistort-and-rectify maps built once on the host, cv::remap INTER_LINEAR on the device.
//
// The maps are built in double with the host libm (CUDA's atan / sqrt may differ from glibc by an ulp, and the build is not per frame),
// stored as the CV_32F maps the reference keeps, and converted once to the fixed-point form cv::remap derives from float maps:
// X = cvRound(map_x * 32), corner (X >> 5) saturated to short, fraction index (Y & 31) * 32 + (X & 31).  The per-frame kernel is then
// integer-only: dst = (sum of w * p + 2^14) >> 15 with the 1024 x 4 bilinear weight table, taps outside the source read 0.
#include "common.cuh"

#include <cmath>
#include <cstdint>
#include <new>
#include <vector>

namespace b200 {
namespace rectify {

constexpr int kThreadsX = 32, kThreadsY = 8, kPxPerThread = 4;  // a CTA owns a 128 x 8 output tile
constexpr int kMaxSide = 32766;                                 // the fixed-point corner is a short; 32767 must stay outside

// iR = (K_rect R)^-1: product summed left to right, inverse by the 3x3 cofactor formula of cv::invert's small-matrix path.
static bool inv_k_r(const double* Kr, const double* R, double* iR) {
    double A[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) A[3 * i + j] = Kr[3 * i] * R[j] + Kr[3 * i + 1] * R[3 + j] + Kr[3 * i + 2] * R[6 + j];
    auto m = [&](int r, int c) { return A[3 * r + c]; };
    double d = m(0, 0) * (m(1, 1) * m(2, 2) - m(1, 2) * m(2, 1)) - m(0, 1) * (m(1, 0) * m(2, 2) - m(1, 2) * m(2, 0))
               + m(0, 2) * (m(1, 0) * m(2, 1) - m(1, 1) * m(2, 0));
    if (d == 0.0 || !std::isfinite(d)) return false;
    d = 1.0 / d;
    iR[0] = (m(1, 1) * m(2, 2) - m(1, 2) * m(2, 1)) * d;
    iR[1] = (m(0, 2) * m(2, 1) - m(0, 1) * m(2, 2)) * d;
    iR[2] = (m(0, 1) * m(1, 2) - m(0, 2) * m(1, 1)) * d;
    iR[3] = (m(1, 2) * m(2, 0) - m(1, 0) * m(2, 2)) * d;
    iR[4] = (m(0, 0) * m(2, 2) - m(0, 2) * m(2, 0)) * d;
    iR[5] = (m(0, 2) * m(1, 0) - m(0, 0) * m(1, 2)) * d;
    iR[6] = (m(1, 0) * m(2, 1) - m(1, 1) * m(2, 0)) * d;
    iR[7] = (m(0, 1) * m(2, 0) - m(0, 0) * m(2, 1)) * d;
    iR[8] = (m(0, 0) * m(1, 1) - m(0, 1) * m(1, 0)) * d;
    return true;
}

// cv::initUndistortRectifyMap (model 0) / cv::fisheye::initUndistortRectifyMap (model 1), CV_32F.
static bool build_map(int model, int cols, int rows, const double* K, const double* D, int n_dist, const double* R, const double* Kr,
                      float* mx, float* my) {
    double iR[9];
    if (!inv_k_r(Kr, R, iR)) return false;
    const double fx = K[0], fy = K[4], u0 = K[2], v0 = K[5];
    double k[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < n_dist; ++i) k[i] = D[i];
    for (int i = 0; i < rows; ++i) {
        float* rx = mx + (size_t)i * cols;
        float* ry = my + (size_t)i * cols;
        if (model == 0) {
            const double k1 = k[0], k2 = k[1], p1 = k[2], p2 = k[3], k3 = k[4], k4 = k[5], k5 = k[6], k6 = k[7];
            for (int j = 0; j < cols; ++j) {
                const double _x = i * iR[1] + iR[2] + j * iR[0];
                const double _y = i * iR[4] + iR[5] + j * iR[3];
                const double _w = i * iR[7] + iR[8] + j * iR[6];
                const double w = 1.0 / _w, x = _x * w, y = _y * w;
                const double x2 = x * x, y2 = y * y, r2 = x2 + y2, _2xy = 2 * x * y;
                // with 4 or 5 coefficients the denominator is exactly 1
                const double kr = (1 + ((k3 * r2 + k2) * r2 + k1) * r2) / (1 + ((k6 * r2 + k5) * r2 + k4) * r2);
                rx[j] = (float)(fx * (x * kr + p1 * _2xy + p2 * (r2 + 2 * x2)) + u0);
                ry[j] = (float)(fy * (y * kr + p1 * (r2 + 2 * y2) + p2 * _2xy) + v0);
            }
        } else {
            // the fisheye map accumulates the ray per column (the per-pixel product form would round differently)
            double _x = i * iR[1] + iR[2], _y = i * iR[4] + iR[5], _w = i * iR[7] + iR[8];
            for (int j = 0; j < cols; ++j) {
                double u, v;
                if (_w > 0) {
                    const double x = _x / _w, y = _y / _w;
                    const double r = std::sqrt(x * x + y * y);
                    const double th = std::atan(r);
                    const double th2 = th * th, th4 = th2 * th2, th6 = th4 * th2, th8 = th4 * th4;
                    const double thd = th * (1 + k[0] * th2 + k[1] * th4 + k[2] * th6 + k[3] * th8);
                    const double s = (r == 0) ? 1.0 : thd / r;
                    u = fx * x * s + u0;
                    v = fy * y * s + v0;
                } else {
                    u = _x > 0 ? -INFINITY : INFINITY;
                    v = _y > 0 ? -INFINITY : INFINITY;
                }
                rx[j] = (float)u;
                ry[j] = (float)v;
                _x += iR[0];
                _y += iR[3];
                _w += iR[6];
            }
        }
    }
    return true;
}

// cvRound of a float: round half to even; NaN and values outside int give INT_MIN (the x86 conversion's "integer indefinite").
static int32_t cv_round(float v) {
    if (!(v >= -2147483648.0f && v < 2147483648.0f)) return INT32_MIN;
    return (int32_t)std::nearbyint(v);
}
static uint32_t sat_short(int32_t v) { return (uint32_t)(uint16_t)(int16_t)(v < -32768 ? -32768 : v > 32767 ? 32767 : v); }

// Table entry per pixel: .x = corner (sx low 16 bits, sy high 16 bits, both signed), .y = fraction index.
static uint2 fixed_entry(float mx, float my) {
    const int32_t X = cv_round(mx * 32.0f), Y = cv_round(my * 32.0f);
    return make_uint2(sat_short(X >> 5) | (sat_short(Y >> 5) << 16), (uint32_t)((Y & 31) * 32 + (X & 31)));
}

// Bilinear weights cvRound(32768 * (float)(wy * wx)) from float coefficients 1 - a and a, a = k / 32, taps (0,0) (1,0) (0,1) (1,1).
// Every quadruple is exact and sums to 32768, so OpenCV's sum fix-up of initInterTab2D has nothing to do; the build checks it.
static bool weight_table(ushort4* tab) {
    for (int fy = 0; fy < 32; ++fy)
        for (int fx = 0; fx < 32; ++fx) {
            const float ay = fy / 32.0f, ax = fx / 32.0f;
            const float cy[2] = {1.0f - ay, ay}, cx[2] = {1.0f - ax, ax};
            int32_t w[4];
            for (int a = 0; a < 2; ++a)
                for (int b = 0; b < 2; ++b) w[2 * a + b] = cv_round((float)(cy[a] * cx[b]) * 32768.0f);
            if (w[0] + w[1] + w[2] + w[3] != 32768) return false;
            tab[fy * 32 + fx] = make_ushort4((unsigned short)w[0], (unsigned short)w[1], (unsigned short)w[2], (unsigned short)w[3]);
        }
    return true;
}

template <int C>
__device__ __forceinline__ void gather(const unsigned char* __restrict__ s, size_t pitch, int cols, int rows, uint2 e, const ushort4 w,
                                       unsigned char* px) {
    const int sx = (int)(short)(e.x & 0xffffu), sy = (int)(short)(e.x >> 16);
    const bool x0 = (unsigned)sx < (unsigned)cols, x1 = (unsigned)(sx + 1) < (unsigned)cols;
    const bool y0 = (unsigned)sy < (unsigned)rows, y1 = (unsigned)(sy + 1) < (unsigned)rows;
    const unsigned char* r0 = s + (ptrdiff_t)sy * (ptrdiff_t)pitch + (ptrdiff_t)sx * C;
    const unsigned char* r1 = r0 + pitch;
#pragma unroll
    for (int c = 0; c < C; ++c) {
        int acc = 1 << 14;
        if (y0 && x0) acc += (int)w.x * __ldg(r0 + c);
        if (y0 && x1) acc += (int)w.y * __ldg(r0 + C + c);
        if (y1 && x0) acc += (int)w.z * __ldg(r1 + c);
        if (y1 && x1) acc += (int)w.w * __ldg(r1 + C + c);
        px[c] = (unsigned char)(acc >> 15);  // weights sum to 32768: the result is in [0, 255]
    }
}

// grid (ceil(cols / 128), ceil(rows / 8), 2 eyes); thread = 4 consecutive output pixels of one row.  The CTA reads its table entries
// once and loops over the batch's frames, so the table crosses HBM once per batch.  store: 0 bytes, 1 32-bit words, 2 128-bit (C = 4).
template <int C>
__global__ void __launch_bounds__(kThreadsX * kThreadsY) remap_kernel(const uint2* __restrict__ tab, size_t tab_pitch, size_t tab_eye,
                                                                       const ushort4* __restrict__ wtab, const unsigned char* src_l,
                                                                       const unsigned char* src_r, size_t src_pitch, size_t src_fs,
                                                                       unsigned char* out_l, unsigned char* out_r, size_t out_pitch,
                                                                       size_t out_fs, int cols, int rows, int batch, int store) {
    __shared__ ushort4 w_s[1024];
    for (int k = threadIdx.y * kThreadsX + threadIdx.x; k < 1024; k += kThreadsX * kThreadsY) w_s[k] = wtab[k];
    __syncthreads();
    const int eye = blockIdx.z;
    const int x0 = (blockIdx.x * kThreadsX + threadIdx.x) * kPxPerThread, y = blockIdx.y * kThreadsY + threadIdx.y;
    if (y >= rows || x0 >= cols) return;
    const int n = min(kPxPerThread, cols - x0);
    // rows of the table are padded to a multiple of 4 entries (32 bytes): two 128-bit loads per thread
    const uint4* t = reinterpret_cast<const uint4*>(tab + eye * tab_eye + (size_t)y * tab_pitch + x0);
    const uint4 ta = __ldg(t), tb = __ldg(t + 1);
    const uint2 e[4] = {make_uint2(ta.x, ta.y), make_uint2(ta.z, ta.w), make_uint2(tb.x, tb.y), make_uint2(tb.z, tb.w)};
    ushort4 w[4];
#pragma unroll
    for (int p = 0; p < 4; ++p) w[p] = w_s[e[p].y];
    const unsigned char* src = eye ? src_r : src_l;
    unsigned char* out = (eye ? out_r : out_l) + (size_t)y * out_pitch + (size_t)x0 * C;
    for (int f = 0; f < batch; ++f) {
        const unsigned char* s = src + (size_t)f * src_fs;
        unsigned char* o = out + (size_t)f * out_fs;
        alignas(16) unsigned char px[4 * C];
#pragma unroll
        for (int p = 0; p < 4; ++p) gather<C>(s, src_pitch, cols, rows, e[p], w[p], px + p * C);
        if constexpr (C == 4) {
            if (n == 4 && store == 2) {
                *reinterpret_cast<uint4*>(o) = *reinterpret_cast<const uint4*>(px);
                continue;
            }
        }
        if (n == 4 && store) {
#pragma unroll
            for (int k = 0; k < C; ++k) reinterpret_cast<uint32_t*>(o)[k] = reinterpret_cast<const uint32_t*>(px)[k];
        } else {
#pragma unroll
            for (int k = 0; k < 4 * C; ++k)
                if (k < n * C) o[k] = px[k];
        }
    }
}

}  // namespace rectify
}  // namespace b200

struct b200_rectifier_s {
    b200_rectifier_params_t prm;
    cudaStream_t own_stream = nullptr, stream = nullptr;
    std::vector<float> map[2][2];  // [eye][x / y], rows x cols
    uint2* d_tab = nullptr;        // [eye][rows][tab_pitch]
    ushort4* d_w = nullptr;        // 1024 weight quadruples
    size_t tab_pitch = 0;          // entries per row (multiple of 4)
};

namespace {

int launch_remap(b200_rectifier_s* h, int channels, const unsigned char* l, const unsigned char* r, size_t src_pitch, size_t src_fs,
                 unsigned char* ol, unsigned char* orr, size_t out_pitch, size_t out_fs, int batch) {
    using namespace b200::rectify;
    const int cols = h->prm.cols, rows = h->prm.rows;
    const bool word = !(((uintptr_t)ol | (uintptr_t)orr | out_pitch | (batch > 1 ? out_fs : 0)) & 3);
    const bool quad = channels == 4 && !(((uintptr_t)ol | (uintptr_t)orr | out_pitch | (batch > 1 ? out_fs : 0)) & 15);
    const int store = quad ? 2 : word ? 1 : 0;
    const dim3 grid(b200::ceil_div(cols, kThreadsX * kPxPerThread), b200::ceil_div(rows, kThreadsY), 2), block(kThreadsX, kThreadsY);
    const size_t tab_eye = h->tab_pitch * (size_t)rows;
#define B200_REMAP(C)                                                                                                                     \
    remap_kernel<C><<<grid, block, 0, h->stream>>>(h->d_tab, h->tab_pitch, tab_eye, h->d_w, l, r, src_pitch, src_fs, ol, orr, out_pitch, \
                                                   out_fs, cols, rows, batch, store)
    if (channels == 1) B200_REMAP(1);
    else if (channels == 3) B200_REMAP(3);
    else B200_REMAP(4);
#undef B200_REMAP
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

void free_rectifier(b200_rectifier_s* h) {
    if (h->d_tab) cudaFree(h->d_tab);
    if (h->d_w) cudaFree(h->d_w);
    if (h->own_stream) cudaStreamDestroy(h->own_stream);
    delete h;
}

}  // namespace

extern "C" {

int b200_rectifier_create(const b200_rectifier_params_t* p, b200_rectifier_t* out) {
    B200_RANGE("b200:rectify:create");
    using namespace b200::rectify;
    if (!p || !out) {
        b200::set_error("b200_rectifier_create: null argument");
        return B200_ERR_INVALID;
    }
    if ((p->model != 0 && p->model != 1) || p->cols < 1 || p->rows < 1 || p->cols > kMaxSide || p->rows > kMaxSide) {
        b200::set_error("b200_rectifier_create: model must be 0 (perspective) or 1 (fisheye) and the size within 1..%d (got model %d, %d x %d)",
                        kMaxSide, p->model, p->cols, p->rows);
        return B200_ERR_INVALID;
    }
    for (int eye = 0; eye < 2; ++eye) {
        const int n = p->n_dist[eye];
        if (p->model == 0 ? (n != 4 && n != 5 && n != 8) : n != 4) {
            b200::set_error("b200_rectifier_create: %d distortion coefficients for the %s model (perspective: 4, 5 or 8; fisheye: 4)", n,
                            p->model == 0 ? "perspective" : "fisheye");
            return B200_ERR_INVALID;
        }
    }
    ushort4 wtab[1024];
    if (!weight_table(wtab)) {
        b200::set_error("b200_rectifier_create: bilinear weight table does not sum to 32768");
        return B200_ERR_INVALID;
    }
    int rc = b200::require_device(p->device);
    if (rc) return rc;
    b200_rectifier_s* h = new (std::nothrow) b200_rectifier_s();
    if (!h) return B200_ERR_INVALID;
    h->prm = *p;
    const size_t cols = (size_t)p->cols, rows = (size_t)p->rows;
    h->tab_pitch = b200::round_up(cols, (size_t)4);
    std::vector<uint2> tab(2 * h->tab_pitch * rows, make_uint2(0x80008000u, 0u));  // padding: corner (-32768, -32768), outside
    for (int eye = 0; eye < 2; ++eye) {
        h->map[eye][0].resize(cols * rows);
        h->map[eye][1].resize(cols * rows);
        if (!build_map(p->model, p->cols, p->rows, p->K[eye], p->D[eye], p->n_dist[eye], p->R[eye], p->K_rect, h->map[eye][0].data(),
                       h->map[eye][1].data())) {
            delete h;
            b200::set_error("b200_rectifier_create: K_rect * R of eye %d is singular", eye);
            return B200_ERR_INVALID;
        }
        for (size_t i = 0; i < rows; ++i)
            for (size_t j = 0; j < cols; ++j)
                tab[(eye * rows + i) * h->tab_pitch + j] = fixed_entry(h->map[eye][0][i * cols + j], h->map[eye][1][i * cols + j]);
    }
    cudaError_t e = cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaMalloc((void**)&h->d_tab, sizeof(uint2) * tab.size());
    if (e == cudaSuccess) e = cudaMalloc((void**)&h->d_w, sizeof(wtab));
    if (e == cudaSuccess) e = cudaMemcpy(h->d_tab, tab.data(), sizeof(uint2) * tab.size(), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(h->d_w, wtab, sizeof(wtab), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        free_rectifier(h);
        return b200::cuda_fail(e, "b200_rectifier_create", __FILE__, __LINE__);
    }
    h->stream = h->own_stream;
    *out = h;
    return B200_OK;
}

int b200_rectifier_destroy(b200_rectifier_t h) {
    if (!h) return B200_OK;
    cudaSetDevice(h->prm.device);
    cudaStreamSynchronize(h->stream);
    free_rectifier(h);
    return B200_OK;
}

int b200_rectifier_set_stream(b200_rectifier_t h, void* stream, int use_own) {
    if (!h) return B200_ERR_INVALID;
    B200_CUDA(cudaSetDevice(h->prm.device));
    B200_CUDA(cudaStreamSynchronize(h->stream));
    h->stream = use_own ? h->own_stream : (cudaStream_t)stream;
    return B200_OK;
}

int b200_rectifier_maps(b200_rectifier_t h, int eye, float* map_x, float* map_y) {
    if (!h || (eye != 0 && eye != 1) || !map_x || !map_y) {
        b200::set_error("b200_rectifier_maps: handle, eye 0 / 1 and both outputs are required");
        return B200_ERR_INVALID;
    }
    std::memcpy(map_x, h->map[eye][0].data(), sizeof(float) * h->map[eye][0].size());
    std::memcpy(map_y, h->map[eye][1].data(), sizeof(float) * h->map[eye][1].size());
    return B200_OK;
}

int b200_stereo_rectify_device(b200_rectifier_t h, int channels, const void* d_left, const void* d_right, size_t src_pitch, size_t src_frame_stride,
                               void* d_out_left, void* d_out_right, size_t out_pitch, size_t out_frame_stride, int batch) {
    B200_RANGE("b200:rectify:device");
    if (!h) {
        b200::set_error("b200_stereo_rectify_device: null handle");
        return B200_ERR_INVALID;
    }
    if (batch == 0) return B200_OK;
    const size_t row = (size_t)h->prm.cols * (size_t)channels, rows = (size_t)h->prm.rows;
    const size_t src_frame = src_pitch * (rows - 1) + row, out_frame = out_pitch * (rows - 1) + row;
    if (batch < 0 || (channels != 1 && channels != 3 && channels != 4) || !d_left || !d_right || !d_out_left || !d_out_right || src_pitch < row
        || out_pitch < row || (batch > 1 && (src_frame_stride < src_frame || out_frame_stride < out_frame))) {
        b200::set_error("b200_stereo_rectify_device: channels 1, 3 or 4, non-null frames, pitches >= cols * channels, frame strides >= one "
                        "frame (batch %d, channels %d, pitches %zu / %zu)", batch, channels, src_pitch, out_pitch);
        return B200_ERR_INVALID;
    }
    B200_CUDA(cudaSetDevice(h->prm.device));
    return launch_remap(h, channels, (const unsigned char*)d_left, (const unsigned char*)d_right, src_pitch, src_frame_stride,
                        (unsigned char*)d_out_left, (unsigned char*)d_out_right, out_pitch, out_frame_stride, batch);
}

int b200_stereo_rectify(b200_rectifier_t h, int channels, const uint8_t* left, size_t left_pitch, const uint8_t* right, size_t right_pitch,
                        uint8_t* out_left, size_t out_left_pitch, uint8_t* out_right, size_t out_right_pitch) {
    B200_RANGE("b200:rectify:host");
    const size_t row = h ? (size_t)h->prm.cols * (size_t)channels : 0;
    if (!h || (channels != 1 && channels != 3 && channels != 4) || !left || !right || !out_left || !out_right || left_pitch < row
        || right_pitch < row || out_left_pitch < row || out_right_pitch < row) {
        b200::set_error("b200_stereo_rectify: channels 1, 3 or 4, non-null frames and pitches >= cols * channels");
        return B200_ERR_INVALID;
    }
    B200_CUDA(cudaSetDevice(h->prm.device));
    const size_t rows = (size_t)h->prm.rows, pitch = b200::round_up(row, (size_t)16), frame = b200::round_up(pitch * rows, (size_t)256);
    unsigned char* d = nullptr;
    B200_CUDA(cudaMallocAsync((void**)&d, 4 * frame, h->stream));
    cudaStream_t st = h->stream;
    cudaError_t e = cudaMemcpy2DAsync(d, pitch, left, left_pitch, row, rows, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpy2DAsync(d + frame, pitch, right, right_pitch, row, rows, cudaMemcpyHostToDevice, st);
    int rc = B200_OK;
    if (e == cudaSuccess) rc = launch_remap(h, channels, d, d + frame, pitch, 0, d + 2 * frame, d + 3 * frame, pitch, 0, 1);
    if (e == cudaSuccess && rc == B200_OK) e = cudaMemcpy2DAsync(out_left, out_left_pitch, d + 2 * frame, pitch, row, rows, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess && rc == B200_OK) e = cudaMemcpy2DAsync(out_right, out_right_pitch, d + 3 * frame, pitch, row, rows, cudaMemcpyDeviceToHost, st);
    cudaFreeAsync(d, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return b200::cuda_fail(e, "b200_stereo_rectify", __FILE__, __LINE__);
    return rc;
}

}  // extern "C"
