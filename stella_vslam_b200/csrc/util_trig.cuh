// util_trig.cuh -- util::cos / util::sin (util/trigonometric.h:11-46) as device functions, shared by the rBRIEF orientation
// (orb_kernels.cu) and the PnP solver's max_cos_errors_ (pnp_kernels.cu).  fp32 with explicit round-to-nearest intrinsics.
#pragma once

namespace b200 {

__device__ __forceinline__ float poly_cos(float v) {
    const float v2 = __fmul_rn(v, v);
    return __fadd_rn(0.99940307f, __fmul_rn(v2, __fadd_rn(-0.49558072f, __fmul_rn(0.03679168f, v2))));
}
__device__ __forceinline__ float util_cos(float v) {
    const float PI = 3.14159265358979f;
    const float PI_2 = __fdiv_rn(PI, 2.0f), TWO_PI = __fmul_rn(2.0f, PI);
    const float INV_TWO_PI = __fdiv_rn(1.0f, TWO_PI), THREE_PI_2 = __fmul_rn(3.0f, PI_2);
    v = __fsub_rn(v, __fmul_rn((float)__float2int_rd(__fmul_rn(v, INV_TWO_PI)), TWO_PI));
    v = (0.0f < v) ? v : -v;
    if (v < PI_2) return poly_cos(v);
    if (v < PI) return -poly_cos(__fsub_rn(PI, v));
    if (v < THREE_PI_2) return -poly_cos(__fsub_rn(v, PI));
    return poly_cos(__fsub_rn(TWO_PI, v));
}
__device__ __forceinline__ float util_sin(float v) {
    const float PI_2 = __fdiv_rn(3.14159265358979f, 2.0f);
    return util_cos(__fsub_rn(PI_2, v));
}

}  // namespace b200
