/* rectify_oracle.c -- CPU restatement of util::stereo_rectifier (test infrastructure, compiled by tests/rectify_oracle.py).
 *
 *   cv::initUndistortRectifyMap           (perspective, CV_32F maps; 4, 5 or 8 distortion coefficients)
 *   cv::fisheye::initUndistortRectifyMap  (4 coefficients; rays behind the camera map to -inf)
 *   the fixed-point form cv::remap derives from float maps (INTER_BITS = 5)
 *   cv::remap INTER_LINEAR, BORDER_CONSTANT 0, 8-bit data with 1, 3 or 4 channels
 *
 * Everything is written out independently of the library: maps in double, stored as float; remap in integers only. */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

/* iR = (K_rect * R)^-1: the product summed left to right, the inverse by the 3x3 cofactor formula of cv::invert's small-matrix
 * path (determinant expanded along the first row). */
static int inv_k_r(const double* Kr, const double* R, double* iR) {
    double A[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) A[3 * i + j] = Kr[3 * i] * R[j] + Kr[3 * i + 1] * R[3 + j] + Kr[3 * i + 2] * R[6 + j];
#define M(r, c) A[3 * (r) + (c)]
    double d = M(0, 0) * (M(1, 1) * M(2, 2) - M(1, 2) * M(2, 1)) - M(0, 1) * (M(1, 0) * M(2, 2) - M(1, 2) * M(2, 0))
               + M(0, 2) * (M(1, 0) * M(2, 1) - M(1, 1) * M(2, 0));
    if (d == 0.0) return -1;
    d = 1.0 / d;
    iR[0] = (M(1, 1) * M(2, 2) - M(1, 2) * M(2, 1)) * d;
    iR[1] = (M(0, 2) * M(2, 1) - M(0, 1) * M(2, 2)) * d;
    iR[2] = (M(0, 1) * M(1, 2) - M(0, 2) * M(1, 1)) * d;
    iR[3] = (M(1, 2) * M(2, 0) - M(1, 0) * M(2, 2)) * d;
    iR[4] = (M(0, 0) * M(2, 2) - M(0, 2) * M(2, 0)) * d;
    iR[5] = (M(0, 2) * M(1, 0) - M(0, 0) * M(1, 2)) * d;
    iR[6] = (M(1, 0) * M(2, 1) - M(1, 1) * M(2, 0)) * d;
    iR[7] = (M(0, 1) * M(2, 0) - M(0, 0) * M(2, 1)) * d;
    iR[8] = (M(0, 0) * M(1, 1) - M(0, 1) * M(1, 0)) * d;
#undef M
    return 0;
}

/* model 0: perspective (n_dist 4, 5 or 8: k1 k2 p1 p2 [k3 [k4 k5 k6]]); model 1: fisheye (n_dist 4: k1..k4).
 * K, R, K_rect: row-major 3x3.  Returns 0, or -1 for an unsupported model / coefficient count / singular K_rect * R. */
int orc_rect_map(int model, int cols, int rows, const double* K, const double* D, int n_dist, const double* R, const double* K_rect,
                 float* map_x, float* map_y) {
    double iR[9];
    if (model == 0 && n_dist != 4 && n_dist != 5 && n_dist != 8) return -1;
    if (model == 1 && n_dist != 4) return -1;
    if (model != 0 && model != 1) return -1;
    if (inv_k_r(K_rect, R, iR)) return -1;
    const double fx = K[0], fy = K[4], u0 = K[2], v0 = K[5];
    double k[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < n_dist; ++i) k[i] = D[i];
    for (int i = 0; i < rows; ++i) {
        float* mx = map_x + (size_t)i * cols;
        float* my = map_y + (size_t)i * cols;
        if (model == 0) {
            const double k1 = k[0], k2 = k[1], p1 = k[2], p2 = k[3], k3 = k[4], k4 = k[5], k5 = k[6], k6 = k[7];
            for (int j = 0; j < cols; ++j) {
                const double _x = i * iR[1] + iR[2] + j * iR[0];
                const double _y = i * iR[4] + iR[5] + j * iR[3];
                const double _w = i * iR[7] + iR[8] + j * iR[6];
                const double w = 1.0 / _w, x = _x * w, y = _y * w;
                const double x2 = x * x, y2 = y * y, r2 = x2 + y2, _2xy = 2 * x * y;
                const double kr = (1 + ((k3 * r2 + k2) * r2 + k1) * r2) / (1 + ((k6 * r2 + k5) * r2 + k4) * r2);
                const double u = fx * (x * kr + p1 * _2xy + p2 * (r2 + 2 * x2)) + u0;
                const double v = fy * (y * kr + p1 * (r2 + 2 * y2) + p2 * _2xy) + v0;
                mx[j] = (float)u;
                my[j] = (float)v;
            }
        } else {
            double _x = i * iR[1] + iR[2], _y = i * iR[4] + iR[5], _w = i * iR[7] + iR[8];
            for (int j = 0; j < cols; ++j) {
                double u, v;
                if (_w > 0) {
                    const double x = _x / _w, y = _y / _w;
                    const double r = sqrt(x * x + y * y);
                    const double th = atan(r);
                    const double th2 = th * th, th4 = th2 * th2, th6 = th4 * th2, th8 = th4 * th4;
                    const double thd = th * (1 + k[0] * th2 + k[1] * th4 + k[2] * th6 + k[3] * th8);
                    const double s = (r == 0) ? 1.0 : thd / r;
                    u = fx * x * s + u0;
                    v = fy * y * s + v0;
                } else {  /* behind the camera: an infinity of the sign opposite to the ray's x (y) */
                    u = _x > 0 ? -INFINITY : INFINITY;
                    v = _y > 0 ? -INFINITY : INFINITY;
                }
                mx[j] = (float)u;
                my[j] = (float)v;
                _x += iR[0];
                _y += iR[3];
                _w += iR[6];
            }
        }
    }
    return 0;
}

/* cvRound of a float: round half to even; NaN and values outside int give INT_MIN (the x86 conversion's "integer indefinite"). */
static int32_t cv_round(float v) {
    if (!(v >= -2147483648.0f && v < 2147483648.0f)) return INT32_MIN;
    return (int32_t)rintf(v);
}

static int16_t sat_short(int32_t v) { return (int16_t)(v < -32768 ? -32768 : v > 32767 ? 32767 : v); }

/* Float maps -> (sx, sy) source corner and the fraction index (Y & 31) * 32 + (X & 31), with X = cvRound(map_x * 32). */
void orc_rect_fixed(size_t n, const float* map_x, const float* map_y, int16_t* sxy, uint16_t* frac) {
    for (size_t p = 0; p < n; ++p) {
        const int32_t X = cv_round(map_x[p] * 32.0f), Y = cv_round(map_y[p] * 32.0f);
        sxy[2 * p] = sat_short(X >> 5);
        sxy[2 * p + 1] = sat_short(Y >> 5);
        frac[p] = (uint16_t)((Y & 31) * 32 + (X & 31));
    }
}

/* Bilinear weight table: entry (fy * 32 + fx) = cvRound(32768 * (float)(wy * wx)) for the taps (0,0) (1,0) (0,1) (1,1), with float
 * coefficients 1 - a and a, a = k / 32.  Returns the number of entries whose weights do not sum to 32768. */
int orc_rect_weights(int32_t* tab) {
    int bad = 0;
    for (int fy = 0; fy < 32; ++fy)
        for (int fx = 0; fx < 32; ++fx) {
            const float ay = fy / 32.0f, ax = fx / 32.0f;
            const float cy[2] = {1.0f - ay, ay}, cx[2] = {1.0f - ax, ax};
            int32_t* t = tab + 4 * (fy * 32 + fx);
            int sum = 0;
            for (int a = 0; a < 2; ++a)
                for (int b = 0; b < 2; ++b) sum += t[2 * a + b] = cv_round((float)(cy[a] * cx[b]) * 32768.0f);
            bad += sum != 32768;
        }
    return bad;
}

/* dst (cols x rows, channels interleaved) from src (src_cols x src_rows) at the fixed-point map. */
void orc_remap(int cols, int rows, int channels, const uint8_t* src, size_t src_pitch, int src_cols, int src_rows, const int16_t* sxy,
               const uint16_t* frac, uint8_t* dst, size_t dst_pitch) {
    int32_t tab[4096];
    orc_rect_weights(tab);
    for (int i = 0; i < rows; ++i)
        for (int j = 0; j < cols; ++j) {
            const size_t p = (size_t)i * cols + j;
            const int sx = sxy[2 * p], sy = sxy[2 * p + 1];
            const int32_t* w = tab + 4 * frac[p];
            for (int c = 0; c < channels; ++c) {
                int32_t acc = 0;
                for (int t = 0; t < 4; ++t) {
                    const int x = sx + (t & 1), y = sy + (t >> 1);
                    if (x >= 0 && y >= 0 && x < src_cols && y < src_rows) acc += w[t] * src[(size_t)y * src_pitch + (size_t)x * channels + c];
                }
                const int32_t v = (acc + (1 << 14)) >> 15;
                dst[(size_t)i * dst_pitch + (size_t)j * channels + c] = (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v);
            }
        }
}
