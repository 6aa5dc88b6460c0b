// camera_model.cuh -- the four camera models of b200_camera_intrinsics_t on the device and camera::*::reproject_to_image, shared by
// the extractor's keypoint kernels and tracking chain (orb_kernels.cu) and the initialiser's triangulation (initialize_kernels.cu).
// reproject_to_image is written as plain double arithmetic: every file that includes it is compiled with -fmad=false, so it is
// evaluated as written.
#pragma once

#include "common.cuh"

namespace b200 {
namespace orb {

struct CamModel {
    int model;  // 0 perspective, 1 equirectangular, 2 fisheye, 3 radial division
    double fx, fy, cx, cy, k1, k2, p1, p2, k3, cols, rows, k4, distortion;
};
__host__ __device__ inline CamModel cam_model(const b200_camera_intrinsics_t& c) {
    return CamModel{c.model, c.fx, c.fy, c.cx, c.cy, c.k1, c.k2, c.p1, c.p2, c.k3, c.cols, c.rows, c.k4, c.distortion};
}
// camera::*::reproject_to_image (perspective.cc:130-148, fisheye.cc:169-187, equirectangular.cc:59-73, radial_division.cc:113-133) of
// the world point p under the pose Rt (rot_cw row-major, then trans_cw): pixel (qx, qy), x_right qr, and whether it lies in the image.
__device__ __forceinline__ bool reproject_to_image(const CamModel& cam, double fxb, float min_x, float max_x, float min_y, float max_y, const double* Rt,
                                                   double px, double py, double pz, double& qx, double& qy, float& qr) {
    const double pcx = Rt[0] * px + Rt[1] * py + Rt[2] * pz + Rt[9];
    const double pcy = Rt[3] * px + Rt[4] * py + Rt[5] * pz + Rt[10];
    const double pcz = Rt[6] * px + Rt[7] * py + Rt[8] * pz + Rt[11];
    bool in_image;
    if (cam.model == 1) {
        const double nrm = sqrt(pcx * pcx + pcy * pcy + pcz * pcz);
        const double bx = pcx / nrm, by = pcy / nrm, bz = pcz / nrm;
        const double latitude = -asin(by), longitude = atan2(bx, bz);
        qx = cam.cols * (0.5 + longitude / (2.0 * 3.14159265358979323846));
        qy = cam.rows * (0.5 - latitude / 3.14159265358979323846);
        qr = 0.f;
        in_image = true;
    } else {
        const double z_inv = 1.0 / pcz;
        qx = cam.fx * pcx * z_inv + cam.cx;
        qy = cam.fy * pcy * z_inv + cam.cy;
        qr = (float)(qx - fxb * z_inv);
        if (cam.model == 3)  // radial_division.cc:124-130: inclusive bounds
            in_image = pcz > 0.0 && !(qx < (double)min_x || qx > (double)max_x) && !(qy < (double)min_y || qy > (double)max_y);
        else                 // perspective.cc:146-147, fisheye.cc:184-186: strict bounds
            in_image = pcz > 0.0 && (double)min_x < qx && qx < (double)max_x && (double)min_y < qy && qy < (double)max_y;
    }
    return in_image;
}

}  // namespace orb
}  // namespace b200
