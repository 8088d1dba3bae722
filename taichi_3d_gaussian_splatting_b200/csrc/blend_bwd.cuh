// blend_bwd.cuh -- declarations shared by the two implementations of loop A of the backward
// (blend_bwd.cu: butterfly reduction per (warp, splat); blend_bwd_transposed.cu: splat-per-lane accumulation).
#pragma once
#include "common.cuh"

namespace gsb {

struct BlendBwdParams {
    int H, W, tiles_x;
    const int *tile_start;
    const int *tile_end;
    const int *sorted_vals;
    const float4 *records;
    const float *grad_image;
    const float *acc_alpha;
    const int *last_effective;
    float *accum;      // rows of 12 floats
    float *mag_image;  // (H,W,2)
    unsigned long long *work_counters;  // COUNT instantiation only: [0] (warp, splat) visits, [1] contributing (pixel, splat) pairs
    const float *grad_depth;  // DEPTH instantiation only: (H,W) dL/d depth and the forward's depth output; NULL otherwise
    const float *depth;
    const float *grad_alpha;  // ALPHA instantiation only: (H,W) dL/d pixel_accumulated_alpha; NULL otherwise
};
// gsb200_backward_ext: C = channels, the (N,C) feature rows the forward blended (gathered by scene row
// point_id[in-camera offset]), the (H,W,C) feature-map gradient and the zeroed (N,C) rows dL/df
struct BlendFeatureParams {
    int channels;
    const int *point_id;
    const float *features;
    const float *grad_feature_map;
    float *grad_features;
};
// The parameter block of the feature instantiations (CF > 0) of the transposed kernel.  The other kernels keep
// BlendBwdParams as it is: a larger parameter block changes their register allocation.
struct BlendBwdFeatParams : BlendBwdParams {
    BlendFeatureParams feat;
};
__device__ __forceinline__ BlendFeatureParams feature_params(const BlendBwdParams &) {
    return BlendFeatureParams{0, nullptr, nullptr, nullptr, nullptr};
}
__device__ __forceinline__ BlendFeatureParams feature_params(const BlendBwdFeatParams &p) { return p.feat; }

#ifdef GSB_HOST_EMU  // tests/simt: the kernels compiled as host C++ under a lock-step SIMT emulator
__device__ __forceinline__ float ex2_approx_b(float x) { return exp2f(x); }
__device__ __forceinline__ float rcp_approx(float x) { return 1.0f / x; }
__device__ __forceinline__ float sqrt_approx(float x) { return sqrtf(x); }
#else
__device__ __forceinline__ float ex2_approx_b(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float rcp_approx(float x) {  // MUFU.RCP, <= 1 ulp
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float sqrt_approx(float x) {  // MUFU.RSQ based, ~1 ulp
    float y;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
#endif

int launch_blend_backward_transposed(const BlendBwdParams &p, int tiles, bool exact_exp, bool stats,
                                     cudaStream_t stream, bool depth = false, bool alpha = false,
                                     const BlendFeatureParams *feat = nullptr, bool wrap = false);
int launch_blend_backward_count(const BlendBwdParams &p, int tiles, cudaStream_t stream);

}  // namespace gsb
