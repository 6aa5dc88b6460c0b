/*
 * tests/motion_track_oracle.c -- TEST INFRASTRUCTURE.  CPU restatement of camera::*::reproject_to_image for the four camera models, written
 * from the reference's behaviour independently of the device code:
 *   perspective     camera/perspective.cc:130-148      pinhole projection of the camera-frame point, strict bounds, z > 0
 *   fisheye         camera/fisheye.cc:169-187          the same pinhole formula and strict bounds on the undistorted image
 *   equirectangular camera/equirectangular.cc:59-73    longitude / latitude of the normalised bearing, always inside, x_right = 0
 *   radial division camera/radial_division.cc:113-133  the pinhole formula with inclusive bounds
 * x_right = u - focal_x_baseline / z for the pinhole family.  Compiled without contraction (-ffp-contract=off), so every double
 * operation is rounded as written.
 */
#include <math.h>
#include <stdint.h>

#define MTO_PI 3.14159265358979323846

/* model: 0 perspective, 1 equirectangular, 2 fisheye, 3 radial division.  Rt_cw: rot_cw row-major, then trans_cw.
 * bounds: the camera's float img_bounds_ (min_x, max_x, min_y, max_y).  Out: in_image, reproj (u, v), x_right. */
void mto_reproject(int model, double fx, double fy, double cx, double cy, double fxb, double cols, double rows, const float* bounds, const double* Rt_cw,
                   int n, const double* pos_w, uint8_t* in_image, double* reproj, float* x_right) {
    for (int i = 0; i < n; ++i) {
        const double* p = pos_w + 3 * i;
        const double pc0 = Rt_cw[0] * p[0] + Rt_cw[1] * p[1] + Rt_cw[2] * p[2] + Rt_cw[9];
        const double pc1 = Rt_cw[3] * p[0] + Rt_cw[4] * p[1] + Rt_cw[5] * p[2] + Rt_cw[10];
        const double pc2 = Rt_cw[6] * p[0] + Rt_cw[7] * p[1] + Rt_cw[8] * p[2] + Rt_cw[11];
        if (model == 1) {
            const double norm = sqrt(pc0 * pc0 + pc1 * pc1 + pc2 * pc2);
            const double b0 = pc0 / norm, b1 = pc1 / norm, b2 = pc2 / norm;
            const double latitude = -asin(b1), longitude = atan2(b0, b2);
            reproj[2 * i] = cols * (0.5 + longitude / (2.0 * MTO_PI));
            reproj[2 * i + 1] = rows * (0.5 - latitude / MTO_PI);
            x_right[i] = 0.f;
            in_image[i] = 1;
            continue;
        }
        const double z_inv = 1.0 / pc2;
        const double u = fx * pc0 * z_inv + cx, v = fy * pc1 * z_inv + cy;
        reproj[2 * i] = u;
        reproj[2 * i + 1] = v;
        x_right[i] = (float)(u - fxb * z_inv);
        if (model == 3)
            in_image[i] = pc2 > 0.0 && !(u < bounds[0] || u > bounds[1]) && !(v < bounds[2] || v > bounds[3]);
        else
            in_image[i] = pc2 > 0.0 && bounds[0] < u && u < bounds[1] && bounds[2] < v && v < bounds[3];
    }
}
