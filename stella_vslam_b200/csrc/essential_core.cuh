// essential_core.cuh -- essential_core.h compiled as device code, with explicit round-to-nearest intrinsics.  Include it inside the
// kernel file's namespace, after epnp.cuh and util_trig.cuh and the using-declarations of da / ds / dm / dd, svd_core and
// apply_householder_left.  The ES_* qualifiers stay defined for twoview_core.h, which twoview_kernels.cu includes after this file.
#pragma once

#define ES_FN __device__
#define ES_BIG __device__ __noinline__
#define ES_SQRT(x) __dsqrt_rn(x)
#define ES_MAKE_HOUSEHOLDER(v, len, stride, tau, beta) pnp::make_householder((v), (len), (stride), (tau), (beta))
#include "essential_core.h"
