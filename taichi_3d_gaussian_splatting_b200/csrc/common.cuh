// common.cuh -- shared declarations of libgsb200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/gsb200.h"

#define GSB_TILE_PIXELS (GSB_TILE_WIDTH * GSB_TILE_HEIGHT)

namespace gsb {

// ---- error plumbing (thread-local message, C ABI returns a code)
void set_error(const char *fmt, ...);
#define GSB_CUDA_CHECK(expr)                                                                   \
    do {                                                                                       \
        cudaError_t _e = (expr);                                                               \
        if (_e != cudaSuccess) {                                                               \
            gsb::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__,   \
                           __LINE__);                                                          \
            return GSB_ECUDA;                                                                  \
        }                                                                                      \
    } while (0)

// ---- counters living at the head of the workspace
// CNT_MAX_DEPTH_KEY: largest int32(depth * scale) over the frame's in-camera points (low 32 bits of the slot; the per-point
// kernel atomicMax-es it, the sort derives the number of live depth bits from it)
enum Counter { CNT_M = 0, CNT_K = 1, CNT_OVERFLOW = 2, CNT_MAX_DEPTH_KEY = 4 };
enum Ticket { TICKET_SCAN = 0, TICKET_SORT0 = 1 /* ..+7: one per pass; +8: histogram blocks done */ };

// Per-object pose block in the workspace (20 floats):
//   [0..11]  T_camera_pointcloud 3x4 row-major (R | t)     GP3D:51-62
//   [12..14] camera centre in the pointcloud frame (-R^T t)  UT:495-510
struct PoseBlock {
    float T[12];
    float centre[3];
    float pad[5];
};
static_assert(sizeof(PoseBlock) == 80, "PoseBlock layout");

// Resolved device pointers of one frame's workspace.
struct Workspace {
    long long *counters;
    unsigned int *tickets;
    unsigned long long *scan_state;
    unsigned int *sort_hist;
    unsigned int *sort_state;
    int *tile_start;
    int *tile_end;
    PoseBlock *poses;
    int *point_id;
    int *point_offset;
    int *num_tiles;
    float4 *records;        // 3 float4 per in-camera point
    float *point_in_camera; // 3 floats per in-camera point
    void *keys_a, *keys_b, *keys_c;  // emitted keys (a), sorted keys (b), scratch of the radix passes (c)
    int *vals_a, *vals_b, *vals_c;
    GsbWorkspaceLayout layout;
};

int resolve_workspace(void *base, int64_t bytes, int64_t N, int32_t n_obj, int64_t key_capacity,
                      int32_t H, int32_t W, float far_plane, float depth_scale, uint32_t flags,
                      Workspace *ws);

// ---- stage launchers (each enqueues on `stream`, returns GSB_* code)
struct LensParams;
struct RsParams;
struct BlurParams;
struct DefocusParams;
// lens: the distortion of gsb200_forward_lens (checked there, r2_max set), or NULL for the pinhole kernel; rs: the rolling
// shutter of gsb200_forward_rolling_shutter (checked there), or NULL; filter3d: the (N,) 3D smoothing filter of
// gsb200_forward_filter3d (checked there), or NULL; blur: the exposure motion of gsb200_forward_motion_blur (checked there,
// never together with filter3d), or NULL; defocus: the thin lens of gsb200_forward_defocus (checked there, never together with
// filter3d; a NULL blur is then zero motion), or NULL
int launch_preprocess(const GsbForwardArgs &a, const Workspace &ws, cudaStream_t stream, const LensParams *lens = nullptr,
                      const RsParams *rs = nullptr, const float *filter3d = nullptr, const BlurParams *blur = nullptr,
                      const DefocusParams *defocus = nullptr);
// the pose blocks of n (q, t) pairs (pose_kernel without the per-frame clears)
int launch_pose_blocks(const float *q_pc, const float *t_pc, int n, PoseBlock *poses, cudaStream_t stream);
int launch_sort(const Workspace &ws, int64_t key_capacity, cudaStream_t stream);
int launch_tile_ranges(const Workspace &ws, int64_t key_capacity, int num_tiles, cudaStream_t stream);
int launch_tile_ranges_raw(const long long *keys_i64, int64_t n, int *tile_start, int *tile_end,
                           int num_tiles, cudaStream_t stream);
// ext: the per-Gaussian feature vectors to blend alongside the image (gsb200_forward_ext, checked there), or NULL; wrap: the
// WRAP instantiations of an equirectangular frame (gsb200_forward_equirect)
int launch_blend_forward(const GsbForwardArgs &a, const Workspace &ws, cudaStream_t stream,
                         const GsbExtraFeatureArgs *ext = nullptr, bool wrap = false);
// grad_depth / depth: the (H,W) depth gradient and the forward's depth output (gsb200_backward_aux; transposed
// kernel only), or both NULL.  grad_alpha: the (H,W) gradient of the accumulated alpha (transposed kernel only), or NULL.
// ext: the feature-map gradient and the (N,C) output rows, zeroed by the caller (transposed kernel only), or NULL.
// depth_grad: the accumulator rows carry dL/dz in word 11.  wrap: the WRAP instantiations of the transposed kernel for an
// equirectangular frame (gsb200_backward_equirect; the butterfly kernel has none)
int launch_blend_backward(const GsbBackwardArgs &a, const Workspace &ws, cudaStream_t stream,
                          const float *grad_depth = nullptr, const float *depth = nullptr,
                          const float *grad_alpha = nullptr, const GsbExtraFeatureArgs *ext = nullptr, bool wrap = false);
// gsb200_backward_equirect: the EQUIRECT per-point kernel (dense gradients as launch_backward_points, d uv / d pc and J of the
// panorama, depth r); arguments checked by the caller
int launch_backward_points_equirect(const GsbBackwardArgs &a, const Workspace &ws, cudaStream_t stream, bool depth_grad);
// gsb200_backward_ortho: the ORTHO per-point kernel (dense gradients as launch_backward_points; with pose / intr also the camera
// sums and their finishing kernels, as launch_backward_points_calib; filter3d never with pose or intr); arguments checked by the
// caller
int launch_backward_points_ortho(const GsbBackwardArgs &a, const Workspace &ws, cudaStream_t stream, bool depth_grad,
                                 const GsbPoseGradArgs *pose, const GsbIntrinsicsGradArgs *intr, const float *filter3d);
int launch_backward_points(const GsbBackwardArgs &a, const Workspace &ws, cudaStream_t stream,
                           const long long *skip_flag = nullptr, bool depth_grad = false);
// gsb200_backward_lens: the LENS per-point kernel (dense gradients as launch_backward_points, d uv / d pc and J through the
// lens); arguments checked by the caller
int launch_backward_points_lens(const GsbBackwardArgs &a, const Workspace &ws, cudaStream_t stream, bool depth_grad,
                                const LensParams &lens);
// gsb200_backward_lens_grad: the LENS per-point kernel that also sums the coefficient gradient (per-CTA rows in
// lens_grad.temp), and the finishing kernel; arguments checked by the caller
int launch_backward_points_lens_grad(const GsbBackwardArgs &a, const Workspace &ws, cudaStream_t stream, bool depth_grad,
                                     const LensParams &lens, const GsbLensGradArgs &lens_grad);
// gsb200_backward_lens_calib with pose and / or intrinsics: the LENS per-point kernel that also sums the pose, intrinsics and
// (with lens_grad) coefficient gradients in one pass, and their finishing kernels; arguments checked by the caller
int launch_backward_points_lens_calib(const GsbBackwardArgs &a, const Workspace &ws, cudaStream_t stream, bool depth_grad,
                                      const LensParams &lens, const GsbLensGradArgs *lens_grad, const GsbPoseGradArgs *pose,
                                      const GsbIntrinsicsGradArgs *intr);
// gsb200_backward_rolling_shutter: the RS per-point kernel (lens: NULL for a pinhole), with rs_grad also the motion sums
// (per-CTA rows in rs_grad->temp) and the finishing kernel; arguments checked by the caller
int launch_backward_points_rs(const GsbBackwardArgs &a, const Workspace &ws, cudaStream_t stream, bool depth_grad,
                              const LensParams *lens, const RsParams &rs, const GsbRollingShutterGradArgs *rs_grad);
// gsb200_backward_filter3d: the FILTER per-point kernels (lens: NULL for a pinhole; rs: NULL for a global shutter; dense
// gradients as launch_backward_points, skip_flag likewise); arguments checked by the caller
int launch_backward_points_filter(const GsbBackwardArgs &a, const Workspace &ws, cudaStream_t stream, const long long *skip_flag,
                                  bool depth_grad, const LensParams *lens, const RsParams *rs, const float *filter3d);
// gsb200_backward_motion_blur: the BLUR per-point kernel (lens: NULL for a pinhole; rs: NULL for a global shutter), with
// blur_grad also the motion sums (per-CTA rows in blur_grad->temp) and the rolling-shutter finishing kernel; arguments
// checked by the caller
// defocus (gsb200_backward_defocus): the thin lens of the frame, or NULL; defocus_grad (with defocus, never with blur_grad):
// the (a, rho) sums through the same rows and finishing kernel, the finished row's first two values copied to
// defocus_grad->grad
int launch_backward_points_blur(const GsbBackwardArgs &a, const Workspace &ws, cudaStream_t stream, bool depth_grad,
                                const LensParams *lens, const RsParams *rs, const BlurParams &blur,
                                const GsbMotionBlurGradArgs *blur_grad, const DefocusParams *defocus = nullptr,
                                const GsbDefocusGradArgs *defocus_grad = nullptr);
// gsb200_filter3d_from_views (csrc/filter3d.cu; arguments checked by the caller)
int launch_filter3d_from_views(const GsbFilter3dViewsArgs &a, cudaStream_t stream);
// gsb200_backward_pose: the POSE per-point kernel (dense gradients as launch_backward_points, plus the per-CTA pose sums
// in pose.temp) and the per-object finishing kernel; arguments checked by the caller
int launch_backward_points_pose(const GsbBackwardArgs &a, const Workspace &ws, cudaStream_t stream, bool depth_grad,
                                const GsbPoseGradArgs &pose);
// gsb200_backward_calib with intrinsics: the INTR per-point kernel (with the pose sums as well when `pose` is set, in the
// same pass) and the finishing kernels; arguments checked by the caller
int launch_backward_points_calib(const GsbBackwardArgs &a, const Workspace &ws, cudaStream_t stream, bool depth_grad,
                                 const GsbPoseGradArgs *pose, const GsbIntrinsicsGradArgs &intr);
int launch_adam_step(float *param, const float *grad, float *exp_avg, float *exp_avg_sq, long long n, double lr, double beta1,
                     double beta2, double eps, int step, const long long *skip_flag, cudaStream_t stream);
int launch_expand_view_gradients(const GsbExpandArgs &a, cudaStream_t stream);
// MCMC densification (csrc/mcmc.cu); skip_flag as in launch_adam_step
int launch_mcmc_regulariser(const float *features, const int8_t *invalid_mask, float *grad_features, long long N,
                            long long num_valid, float lambda_opacity, float lambda_scale, float *terms_out, void *temp,
                            const long long *skip_flag, cudaStream_t stream);
int launch_mcmc_noise(float *pointcloud, const float *features, const int8_t *invalid_mask, long long N, float noise_scale,
                      float gate_k, float min_opacity, unsigned long long seed, long long step, const long long *skip_flag,
                      cudaStream_t stream);
// supervision_loss.cu: the pre-pass returns the image and ground truth the image loss must read (composited or the inputs)
int launch_supervision_pre(const GsbSupervisionArgs &s, const float *image, const float *gt, const float *alpha,
                           const float *depth, int H, int W, cudaStream_t stream, const float **loss_image,
                           const float **loss_gt);
int launch_supervision_post(const GsbSupervisionArgs &s, const float *image, const float *gt, const float *alpha,
                            const float *depth, int H, int W, const float *grad_image, const float *image_loss,
                            cudaStream_t stream);
// feature_loss.cu: both passes of the feature term (arguments checked by gsb200_train_step_ext)
int launch_feature_loss(const GsbFeatureTrainArgs &x, int H, int W, cudaStream_t stream);
// Per-pixel loss weights (csrc/robust_loss.cu); arguments checked by the caller.  pre: w and x' from the image the loss
// reads; post: dL/dx' -> dL/dx in place, and the stats
int launch_robust_pre(const GsbRobustLossArgs &r, const float *image, const float *gt, int H, int W, cudaStream_t stream);
int launch_robust_post(const GsbRobustLossArgs &r, const float *image, int H, int W, float *grad, cudaStream_t stream);
// appearance.cu: the bilateral-grid slice, its backward (+ the TV term when tv_out is set; arguments checked by the caller)
int launch_bilateral_grid_forward(const float *image, const float *grid, int H, int W, int gx, int gy, int gz, float *out,
                                  cudaStream_t stream);
int launch_bilateral_grid_backward(const float *image, const float *grid, int H, int W, int gx, int gy, int gz,
                                   const float *grad_out, float *grad_in, float *grad_grid, void *temp, float tv_weight,
                                   float *tv_out, cudaStream_t stream);
int launch_blend_forward_count(const GsbForwardArgs &a, const Workspace &ws, unsigned long long *counters_dev,
                               cudaStream_t stream);
int launch_blend_backward_work(const GsbBackwardArgs &a, const Workspace &ws, unsigned long long *counters_dev,
                               cudaStream_t stream);

int sort_radix_bits(int bits);
int sort_pairs_device(const void *keys_in, const int *vals_in, void *keys_out, int *vals_out,
                      const long long *n_dev, int64_t n_capacity, int key_bytes, int depth_bits, int end_bit,
                      const int *max_depth_key /*device or NULL*/, unsigned int *hist /*8*256, zeroed*/,
                      unsigned int *state /*cleared by the sort*/, unsigned int *tickets /*9, zeroed*/, void *tmp_keys,
                      int *tmp_vals, cudaStream_t stream);

#ifndef GSB_SORT_ITEMS
#define GSB_SORT_ITEMS 12
#endif
#ifndef GSB_SORT_MIN_BLOCKS
#define GSB_SORT_MIN_BLOCKS 3
#endif
constexpr int SORT_BLOCK_THREADS = 256;
constexpr int SORT_ITEMS_PER_THREAD = GSB_SORT_ITEMS;
constexpr int SORT_TILE = SORT_BLOCK_THREADS * SORT_ITEMS_PER_THREAD;  // 3072 keys per CTA
#ifndef GSB_SCAN_THREADS
#define GSB_SCAN_THREADS 128
#endif
constexpr int SCAN_BLOCK_THREADS = GSB_SCAN_THREADS;

// ---- per-warp culling shared by the forward and backward blend kernels.
// A CTA renders a 16x16 tile with 8 warps; warp w owns the 8x4 pixel patch at ((w & 1) * 8, (w >> 1) * 4).
// When a batch of splats is staged into shared memory the loading thread computes, for its splat, which
// of the 8 patches it can reach with alpha >= 1/255: alpha = exp(-q/2) * rescale * opacity >= 1/255 needs
// q(d) = d^T conic d <= t2 = 2 ln(255 * rescale * opacity).  A patch is kept iff the minimum of the convex
// quadratic q over the rectangle spanned by the patch's pixel centres is <= t2 (0 if the splat centre is
// inside; otherwise attained on one of the four edges, a clamped 1-D minimisation each).  The test is
// conservative (t2 padded by 0.2 % + 1e-3; degenerate or NaN conics keep every patch), so it never
// changes a result -- it only lets a warp skip splats none of its 32 pixels can see.
#if defined(__CUDACC__) || defined(GSB_HOST_EMU)
#ifdef GSB_HOST_EMU
// tests/simt compiles the blend-backward kernels as host C++ under a lock-step SIMT emulator (simt_emu.h): "shared
// space addresses" are 32-bit offsets from an anchor inside the emulator's image, the approximations are libm calls.
template <int BYTE_OFFSET>
inline float4 lds128(unsigned int saddr) {
    return *reinterpret_cast<const float4 *>(simt_emu::smem_anchor() + (long long)(int)saddr + BYTE_OFFSET);
}
inline unsigned int smem_u32(const void *p) {
    return (unsigned int)(int)(reinterpret_cast<const char *>(p) - simt_emu::smem_anchor());
}
inline float rcp_fast(float x) { return 1.0f / x; }
#else
// 128-bit shared-memory load from an explicit shared-space address (keeps the address arithmetic of the
// blend inner loops to one IMAD instead of a generic->shared window computation per access).
template <int BYTE_OFFSET>
__device__ __forceinline__ float4 lds128(unsigned int saddr) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4+%5];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "r"(saddr), "n"(BYTE_OFFSET));
    return v;
}
// Shared-space address of a __shared__ object, made opaque so that the compiler keeps it in a register
// instead of re-deriving it (S2R SR_CgaCtaId + LEA chain) inside the inner loops.
__device__ __forceinline__ unsigned int smem_u32(const void *p) {
    unsigned int a = (unsigned int)__cvta_generic_to_shared(p);
    asm volatile("" : "+r"(a));
    return a;
}
#endif

// Reach test of one splat: can alpha = exp(-q/2) * ro reach 1/255 anywhere in a rectangle of pixel centres?
// q(d) = d^T conic d <= t2 = 2 ln(255 ro) (padded by 0.2 % + 1e-3).  `mode`: 0 = never (ro too small),
// 1 = test rectangles with rect_reachable(), 2 = always (NaN / degenerate conic: keep the reference behaviour).
// The arithmetic uses explicit FMAs and approximate reciprocals: it only has to be conservative, not exact.
struct SplatReach {
    float a, b2, c;        // conic a, 2b, c
    float nb_ic, nb_ia;    // -b / c, -b / a  (1-D minimisers along vertical / horizontal edges)
    float t2;
    int mode;
};
#ifndef GSB_HOST_EMU
__device__ __forceinline__ float rcp_fast(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
#endif
__device__ __forceinline__ float quad_form(const SplatReach &r, float dx, float dy) {
    return fmaf(dx, fmaf(r.b2, dy, r.a * dx), r.c * dy * dy);
}
__device__ __forceinline__ SplatReach make_splat_reach(float a, float b, float c, float rescale_times_opacity) {
    SplatReach r;
    r.a = a; r.b2 = 2.0f * b; r.c = c;
    const float ro = rescale_times_opacity;
    r.nb_ic = -b * rcp_fast(c);
    r.nb_ia = -b * rcp_fast(a);
    r.t2 = fmaf(2.0f * 1.002f, __logf(fmaxf(255.0f * ro, 1.0f)), 1e-3f);
    const float det = a * c - b * b;
    if (!(ro == ro) || !(det > 0.0f) || !(a > 0.0f) || !(c > 0.0f)) r.mode = 2;
    else if (ro < (1.0f / 255.0f) * 0.999f) r.mode = 0;  // exp(.) <= 1: can never reach 1/255
    else r.mode = 1;
    return r;
}
// Rectangle [X0,X1] x [Y0,Y1] is given RELATIVE to the splat centre.  Minimum of the convex quadratic over the
// rectangle: 0 if the centre is inside, otherwise attained on one of the four edges (clamped 1-D minimisation).
__device__ __forceinline__ bool rect_reachable(const SplatReach &r, float X0, float X1, float Y0, float Y1) {
    if (X0 <= 0.0f && X1 >= 0.0f && Y0 <= 0.0f && Y1 >= 0.0f) return true;
    const float ya = fminf(fmaxf(r.nb_ic * X0, Y0), Y1);
    const float yb = fminf(fmaxf(r.nb_ic * X1, Y0), Y1);
    const float xa = fminf(fmaxf(r.nb_ia * Y0, X0), X1);
    const float xb = fminf(fmaxf(r.nb_ia * Y1, X0), X1);
    const float best = fminf(fminf(quad_form(r, X0, ya), quad_form(r, X1, yb)),
                             fminf(quad_form(r, xa, Y0), quad_form(r, xb, Y1)));
    return !(best > r.t2);  // NaN keeps the rectangle
}

__device__ __forceinline__ unsigned int splat_patch_mask(float u, float v, float a, float b, float c,
                                                         float rescale_times_opacity, float tile_x0,
                                                         float tile_y0) {
    const SplatReach r = make_splat_reach(a, b, c, rescale_times_opacity);
    if (r.mode == 0) return 0u;
    if (r.mode == 2) return 0xFFu;
    unsigned int m = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) {
        // rectangle of the patch's pixel centres, relative to the splat centre
        const float X0 = tile_x0 + 8.0f * (w & 1) + 0.5f - u;
        const float Y0 = tile_y0 + 4.0f * (w >> 1) + 0.5f - v;
        if (rect_reachable(r, X0, X0 + 7.0f, Y0, Y0 + 3.0f)) m |= 1u << w;
    }
    return m;
}
#endif

// ---- alpha of the default (fast) arithmetic path, shared by the forward blend and both backward kernels so that the
// alpha >= 1/255 decision of a (pixel, splat) pair is taken on bit-identical values in both passes.  The staged record
// carries the conic pre-scaled by -log2(e)/2: A = -log2(e)/2 a, B = -log2(e) b, C = -log2(e)/2 c, and ro = rescale * opacity:
//   alpha = 2^(A dx^2 + B dx dy + C dy^2) * ro  =  exp(-(a dx^2 + 2 b dx dy + c dy^2) / 2) * rescale * opacity   (UT:275-284)
#if defined(__CUDACC__) || defined(GSB_HOST_EMU)
constexpr float GSB_L2E = 1.4426950408889634f;
#ifdef GSB_HOST_EMU
__device__ __forceinline__ float ex2_mufu(float x) { return exp2f(x); }
#else
__device__ __forceinline__ float ex2_mufu(float x) {  // one MUFU.EX2; rel. error ~2^-22
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
#endif
__device__ __forceinline__ float fast_alpha(float dx, float dy, float A, float B, float C, float ro) {
    return ex2_mufu(fmaf(dx, fmaf(A, dx, B * dy), (C * dy) * dy)) * ro;
}
// record planes r0 = u v a b, r1 = c rescale opacity depth  ->  staged fast-path planes u v A B | C ro (1 - opacity) depth
__device__ __forceinline__ void fast_planes(const float4 r0, const float4 r1, float4 &s0, float4 &s1) {
    s0 = make_float4(r0.x, r0.y, (-0.5f * GSB_L2E) * r0.z, -GSB_L2E * r0.w);
    s1 = make_float4((-0.5f * GSB_L2E) * r1.x, r1.y * r1.z, 1.0f - r1.z, r1.w);
}
#endif

// ---- lens distortion (gsb200_forward_lens / gsb200_backward_lens; definition in include/gsb200.h).  The per-point forward
// and the per-point backward both call lens_distort, so the position they project to and the Jacobian they differentiate
// agree by construction.
struct LensParams {
    int model;     // GSB_LENS_OPENCV or GSB_LENS_FISHEYE
    float k[5];    // opencv: k1 k2 p1 p2 k3; fisheye: k1 k2 k3 k4 0
    float r2_max;  // r^2 bound of the region where the map does not fold back (inf: unbounded), lens_r2_bound
};
#if defined(__CUDACC__) || defined(GSB_HOST_EMU)
// (xn, yn) -> the displacement (ox, oy) = (xd - xn, yd - yn) and D = d(xd, yd)/d(xn, yn), row-major 2x2.  The callers
// project z (xn + ox, yn + oy, 1) = (x + z ox, y + z oy, z) and form K D, diag(fx, fy) D in the pinhole's expression shapes,
// so that an opencv lens with all coefficients 0 (ox = oy = 0, D = I exactly) reproduces the pinhole path bit for bit.
template <int MODEL>
__device__ __forceinline__ void lens_distort(const float *k, float xn, float yn, float &ox, float &oy, float *D) {
    const float r2 = xn * xn + yn * yn;
    if (MODEL == GSB_LENS_OPENCV) {
        const float k1 = k[0], k2 = k[1], p1 = k[2], p2 = k[3], k3 = k[4];
        const float rad1 = r2 * (k1 + r2 * (k2 + r2 * k3));  // rad - 1
        const float rad = 1.0f + rad1;
        const float drad = k1 + r2 * (2.0f * k2 + r2 * (3.0f * k3));  // d rad / d r^2
        ox = xn * rad1 + 2.0f * p1 * xn * yn + p2 * (r2 + 2.0f * xn * xn);
        oy = yn * rad1 + p1 * (r2 + 2.0f * yn * yn) + 2.0f * p2 * xn * yn;
        const float off = 2.0f * xn * yn * drad + 2.0f * (p1 * xn + p2 * yn);
        D[0] = rad + 2.0f * xn * xn * drad + 2.0f * p1 * yn + 6.0f * p2 * xn;
        D[1] = off;
        D[2] = off;
        D[3] = rad + 2.0f * yn * yn * drad + 6.0f * p1 * yn + 2.0f * p2 * xn;
    } else {
        // s = theta_d / r = A P(theta^2) with A = atan(r) / r, P(t) = 1 + k1 t + k2 t^2 + k3 t^3 + k4 t^4, and
        // D = s I + g (xn, yn)^T (xn, yn) with g = (ds/dr) / r = (A'/r) P + 2 A^2 P'(theta^2) / (1 + r^2).
        // A and A'/r are cancellation-free series for small r (both are even in r).
        float A, Ar;
        if (r2 < 0.04f) {
            A = 1.0f + r2 * (-1.0f / 3.0f + r2 * (1.0f / 5.0f + r2 * (-1.0f / 7.0f + r2 * (1.0f / 9.0f + r2 * (-1.0f / 11.0f)))));
            Ar = -2.0f / 3.0f + r2 * (4.0f / 5.0f + r2 * (-6.0f / 7.0f + r2 * (8.0f / 9.0f + r2 * (-10.0f / 11.0f))));
        } else {
            const float r = sqrtf(r2);
            A = atanf(r) / r;
            Ar = (1.0f / (1.0f + r2) - A) / r2;
        }
        const float t = A * A * r2;  // theta^2
        const float P = 1.0f + t * (k[0] + t * (k[1] + t * (k[2] + t * k[3])));
        const float dP = k[0] + t * (2.0f * k[1] + t * (3.0f * k[2] + t * (4.0f * k[3])));
        const float s = A * P;
        const float g = Ar * P + 2.0f * A * A * dP / (1.0f + r2);
        ox = (s - 1.0f) * xn;
        oy = (s - 1.0f) * yn;
        D[0] = s + g * xn * xn;
        D[1] = g * xn * yn;
        D[2] = D[1];
        D[3] = s + g * yn * yn;
    }
}
// The coefficient gradient of lens_distort at (xn, yn) (gsb200_backward_lens_grad): given gx, gy = dL/d(xd, yd) and
// w00, w01, w11 = dL/dD[0][0], dL/dD[0][1] + dL/dD[1][0], dL/dD[1][1] (D is symmetric in both models), writes
// out[i] = gx dxd/dk_i + gy dyd/dk_i + <dL/dD, dD/dk_i> in LensParams::k's order (fisheye: out[4] = 0).  Both maps are linear
// in the coefficients, so the columns d(xd, yd)/dk and dD/dk are closed forms in (xn, yn) alone:
//   opencv, k_m = k1 k2 k3 (m = 1 2 3): d(xd, yd) = r^2m (xn, yn), dD = r^2m I + 2m r^2(m-1) (xn, yn)^T (xn, yn);
//     p1: d(xd, yd) = (2 xn yn, r^2 + 2 yn^2), dD = [2 yn, 2 xn; 2 xn, 6 yn];  p2: (r^2 + 2 xn^2, 2 xn yn), [6 xn, 2 yn; 2 yn, 2 xn]
//   fisheye, t = theta^2 (j = 1..4): ds/dk_j = A t^j, dg/dk_j = (A'/r) t^j + 2 A^2 j t^(j-1) / (1 + r^2), and with
//     (xd, yd) = s (xn, yn), D = s I + g (xn, yn)^T (xn, yn): d(xd, yd) = ds (xn, yn), dD = ds I + dg (xn, yn)^T (xn, yn).
// A and A'/r are lens_distort's (the same series below r^2 = 0.04).
template <int MODEL>
__device__ __forceinline__ void lens_coefficient_grad(float xn, float yn, float gx, float gy, float w00, float w01, float w11,
                                                      float *out) {
    const float r2 = xn * xn + yn * yn;
    const float pos = gx * xn + gy * yn;                               // (gx, gy) . (xn, yn)
    const float tr = w00 + w11;                                        // <dL/dD, I>
    const float quad = w00 * xn * xn + w01 * xn * yn + w11 * yn * yn;  // <dL/dD, (xn, yn)^T (xn, yn)>
    if (MODEL == GSB_LENS_OPENCV) {
        const float r4 = r2 * r2;
        out[0] = r2 * (pos + tr) + 2.0f * quad;
        out[1] = r4 * (pos + tr) + 4.0f * r2 * quad;
        out[2] = gx * (2.0f * xn * yn) + gy * (r2 + 2.0f * yn * yn) + 2.0f * w00 * yn + 2.0f * w01 * xn + 6.0f * w11 * yn;
        out[3] = gx * (r2 + 2.0f * xn * xn) + gy * (2.0f * xn * yn) + 6.0f * w00 * xn + 2.0f * w01 * yn + 2.0f * w11 * xn;
        out[4] = r4 * r2 * (pos + tr) + 6.0f * r4 * quad;
    } else {
        float A, Ar;
        if (r2 < 0.04f) {
            A = 1.0f + r2 * (-1.0f / 3.0f + r2 * (1.0f / 5.0f + r2 * (-1.0f / 7.0f + r2 * (1.0f / 9.0f + r2 * (-1.0f / 11.0f)))));
            Ar = -2.0f / 3.0f + r2 * (4.0f / 5.0f + r2 * (-6.0f / 7.0f + r2 * (8.0f / 9.0f + r2 * (-10.0f / 11.0f))));
        } else {
            const float r = sqrtf(r2);
            A = atanf(r) / r;
            Ar = (1.0f / (1.0f + r2) - A) / r2;
        }
        const float t = A * A * r2;  // theta^2
        const float c = 2.0f * A * A / (1.0f + r2);
        float tj1 = 1.0f;  // t^(j-1)
#pragma unroll
        for (int j = 1; j <= 4; ++j) {
            const float tj = tj1 * t;
            out[j - 1] = A * tj * (pos + tr) + (Ar * tj + c * (float)j * tj1) * quad;
            tj1 = tj;
        }
        out[4] = 0.0f;
    }
}
#endif

// ---- rolling shutter (gsb200_forward_rolling_shutter / gsb200_backward_rolling_shutter; definition in include/gsb200.h)
struct RsParams {
    float motion[6];  // v (3), w (3)
    float *row_time;  // (N): written by the forward, read by the backward
};
#if defined(__CUDACC__) || defined(GSB_HOST_EMU)
// A = sin(theta)/theta, B = (1 - cos(theta))/theta^2, C = (theta - sin(theta))/theta^3 of theta^2 = t2, by their series below
// t2 = 0.01 (cancellation-free; t2 = 0 gives A = 1, B = 1/2 exactly)
__device__ __forceinline__ void rs_series(float t2, float &A, float &B, float &C) {
    if (t2 < 0.01f) {
        A = 1.0f - (t2 / 6.0f) * (1.0f - t2 / 20.0f);
        B = 0.5f * (1.0f - (t2 / 12.0f) * (1.0f - t2 / 30.0f));
        C = (1.0f / 6.0f) * (1.0f - (t2 / 20.0f) * (1.0f - t2 / 42.0f));
    } else {
        const float th = sqrtf(t2);
        const float s = sinf(th);
        A = s / th;
        B = (1.0f - cosf(th)) / t2;
        C = (th - s) / (t2 * th);
    }
}
// Rd(tau) = exp(tau [w]x) = I + A [p]x + B [p]x^2 with p = tau w, row-major.  w = 0 gives I exactly.
__device__ __forceinline__ void rolling_shutter_rotation(float tau, const float *w, float *R) {
    const float px = tau * w[0], py = tau * w[1], pz = tau * w[2];
    float A, B, C;
    rs_series(px * px + py * py + pz * pz, A, B, C);
    R[0] = 1.0f - B * (py * py + pz * pz); R[1] = B * (px * py) - A * pz;        R[2] = B * (px * pz) + A * py;
    R[3] = B * (px * py) + A * pz;        R[4] = 1.0f - B * (px * px + pz * pz); R[5] = B * (py * pz) - A * px;
    R[6] = B * (px * pz) - A * py;        R[7] = B * (py * pz) + A * px;        R[8] = 1.0f - B * (px * px + py * py);
}
// pc(tau) = Rd pc0 + tau v
__device__ __forceinline__ void rolling_shutter_point(const float *R, float tau, const float *v, const float *pc0, float *pc) {
#pragma unroll
    for (int r = 0; r < 3; ++r) pc[r] = ((R[3 * r] * pc0[0] + R[3 * r + 1] * pc0[1]) + R[3 * r + 2] * pc0[2]) + tau * v[r];
}
// The motion gradient of one in-camera point (gsb200_backward_rolling_shutter with rs_grad): out = (dL/dv, dL/dw) of the
// definition in include/gsb200.h.  gp = dL/dpc, pc0 = W xyz + tw, R = Rd(tau), J the full 2x3 J (row-major), B0, B1 the rows of
// G (J W_eff) Sigma, W the object's rotation (row-major).  dL/dRd = gp pc0^T + 2 J^T [B0; B1] W^T; with A = Rd^T dL/dRd and
// a = (A21 - A12, A02 - A20, A10 - A01) (0-based), dL/dw = tau J_r(tau w)^T a, J_r^T a = a + B (p x a) + C p x (p x a).
__device__ __forceinline__ void rolling_shutter_grad(float tau, const float *w, const float *R, const float *pc0, const float *gp,
                                                     const float *J, const float *B0, const float *B1, const float *W,
                                                     float *out) {
    out[0] = tau * gp[0];
    out[1] = tau * gp[1];
    out[2] = tau * gp[2];
    float h0[3], h1[3];  // [B0; B1] W^T
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        h0[j] = B0[0] * W[3 * j] + B0[1] * W[3 * j + 1] + B0[2] * W[3 * j + 2];
        h1[j] = B1[0] * W[3 * j] + B1[1] * W[3 * j + 1] + B1[2] * W[3 * j + 2];
    }
    float G[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int j = 0; j < 3; ++j) G[3 * r + j] = gp[r] * pc0[j] + 2.0f * (J[r] * h0[j] + J[3 + r] * h1[j]);
    float A[9];  // Rd^T G
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int j = 0; j < 3; ++j) A[3 * r + j] = R[r] * G[j] + R[3 + r] * G[3 + j] + R[6 + r] * G[6 + j];
    const float a0 = A[7] - A[5], a1 = A[2] - A[6], a2 = A[3] - A[1];
    const float px = tau * w[0], py = tau * w[1], pz = tau * w[2];
    float sA, sB, sC;
    rs_series(px * px + py * py + pz * pz, sA, sB, sC);
    const float c0 = py * a2 - pz * a1, c1 = pz * a0 - px * a2, c2 = px * a1 - py * a0;  // p x a
    const float d0 = py * c2 - pz * c1, d1 = pz * c0 - px * c2, d2 = px * c1 - py * c0;  // p x (p x a)
    out[3] = tau * (a0 + sB * c0 + sC * d0);
    out[4] = tau * (a1 + sB * c1 + sC * d1);
    out[5] = tau * (a2 + sB * c2 + sC * d2);
}
#endif

// ---- motion blur (gsb200_forward_motion_blur / gsb200_backward_motion_blur; definition in include/gsb200.h)
struct BlurParams {
    float motion[6];  // v (3), w (3) over the whole exposure
};
#if defined(__CUDACC__) || defined(GSB_HOST_EMU)
// m != 0.  A view with m = 0 takes the un-blurred arithmetic, so it reproduces the kernels without blur bit for bit.
__device__ __forceinline__ bool motion_blur_on(const float *m) {
    return m[0] != 0.0f || m[1] != 0.0f || m[2] != 0.0f || m[3] != 0.0f || m[4] != 0.0f || m[5] != 0.0f;
}
// d = Jp (v + w x pc): the screen displacement of the splat centre over the exposure (dj: the full 2x3 position Jacobian
// d(u, v)/d pc, row-major)
__device__ __forceinline__ void motion_blur_velocity(const float *dj, const float *pc, const float *m, float &d0, float &d1) {
    const float u0 = m[0] + (m[4] * pc[2] - m[5] * pc[1]);
    const float u1 = m[1] + (m[5] * pc[0] - m[3] * pc[2]);
    const float u2 = m[2] + (m[3] * pc[1] - m[4] * pc[0]);
    d0 = (dj[0] * u0 + dj[1] * u1) + dj[2] * u2;
    d1 = (dj[3] * u0 + dj[4] * u1) + dj[5] * u2;
}
// The backward of the blur of one in-camera point.  (s00, s01, s11) = Sigma', (d0, d1) = d, g_alpha = G_a; on entry
// (g00, g01, g11) = G = dL/d(Sigma_d + B), on exit dL/dSigma' = G + G_a/2 (Sigma_d^-1 - (Sigma_d + B)^-1) (the compensation
// c_b); (gd0, gd1) = dL/dd = G d / 6 - G_a/12 (Sigma_d + B)^-1 d.
__device__ __forceinline__ void motion_blur_grad(float s00, float s01, float s11, float d0, float d1, float g_alpha, float &g00,
                                                 float &g01, float &g11, float &gd0, float &gd1) {
    const float a00 = s00 + 0.3f, a11 = s11 + 0.3f;  // Sigma_d
    const float b00 = a00 + (d0 * d0) / 12.0f, b01 = s01 + (d0 * d1) / 12.0f, b11 = a11 + (d1 * d1) / 12.0f;  // Sigma_d + B
    const float ia = 1.0f / (a00 * a11 - s01 * s01), ib = 1.0f / (b00 * b11 - b01 * b01);
    const float i00 = ib * b11, i01 = -ib * b01, i11 = ib * b00;  // (Sigma_d + B)^-1
    const float Gd0 = g00 * d0 + g01 * d1, Gd1 = g01 * d0 + g11 * d1;
    const float Id0 = i00 * d0 + i01 * d1, Id1 = i01 * d0 + i11 * d1;
    gd0 = Gd0 / 6.0f - (g_alpha / 12.0f) * Id0;
    gd1 = Gd1 / 6.0f - (g_alpha / 12.0f) * Id1;
    const float h = 0.5f * g_alpha;
    g00 += h * (ia * a11 - i00);
    g01 += h * (-ia * s01 - i01);
    g11 += h * (ia * a00 - i11);
}
#endif

// ---- defocus (gsb200_forward_defocus / gsb200_backward_defocus; definition in include/gsb200.h)
struct DefocusParams {
    float aperture = 0.0f;       // a, scene units
    float inverse_focus = 0.0f;  // rho = 1 / focus distance
};
#if defined(__CUDACC__) || defined(GSB_HOST_EMU)
// beta = a^2 (rho - 1/z)^2 / 16: the per-axis variance, on the normalised image plane, of the aperture disk's image of a point
// at depth z.  B_d = beta M M^T with M = K[:2,:2] (K[:2,:2] D with a lens).
__device__ __forceinline__ float defocus_variance(const DefocusParams &f, float z) {
    const float e = f.inverse_focus - 1.0f / z;
    return (f.aperture * f.aperture) * (e * e) / 16.0f;
}
// The backward of a blur B (the sum of the motion's and the defocus' terms) of one in-camera point: (s00, s01, s11) = Sigma',
// (b00, b01, b11) = B, g_alpha = G_a; on entry (g00, g01, g11) = G = dL/d(Sigma_d + B), on exit dL/dSigma' = G + G_a/2
// (Sigma_d^-1 - (Sigma_d + B)^-1); (h00, h01, h11) = G_B = dL/dB = G - G_a/2 (Sigma_d + B)^-1, the c_b term included.
__device__ __forceinline__ void blur_cov_grad(float s00, float s01, float s11, float b00, float b01, float b11, float g_alpha,
                                              float &g00, float &g01, float &g11, float &h00, float &h01, float &h11) {
    const float a00 = s00 + 0.3f, a11 = s11 + 0.3f;  // Sigma_d
    const float c00 = a00 + b00, c01 = s01 + b01, c11 = a11 + b11;  // Sigma_d + B
    const float ia = 1.0f / (a00 * a11 - s01 * s01), ib = 1.0f / (c00 * c11 - c01 * c01);
    const float i00 = ib * c11, i01 = -ib * c01, i11 = ib * c00;  // (Sigma_d + B)^-1
    const float h = 0.5f * g_alpha;
    h00 = g00 - h * i00;
    h01 = g01 - h * i01;
    h11 = g11 - h * i11;
    g00 += h * (ia * a11 - i00);
    g01 += h * (-ia * s01 - i01);
    g11 += h * (ia * a00 - i11);
}
#endif

// ---- equirectangular panoramas (gsb200_forward_equirect / gsb200_backward_equirect; definition in include/gsb200.h).
// LENS_EQUIRECT is an internal model code of the per-point kernels' LENS switch and of LensParams::model, never a GsbLensArgs
// value: gsb200_forward_lens keeps refusing every model code it does not know.
constexpr int LENS_EQUIRECT = 0x45510;
#if defined(__CUDACC__) || defined(GSB_HOST_EMU)
// The projection of a camera-frame point: rho = |(x, z)|, r = |pc|, u = fx atan2(x, z) + cx reduced into [0, W),
// v = fy atan2(y, rho) + cy.  Returns whether the point is in view (near < r < far, rho > GSB_EQUIRECT_POLE_EPSILON r; NaN
// fails).
__device__ __forceinline__ bool equirect_project(const float *Kc, int W, float near_plane, float far_plane, const float *pc,
                                                 float &u, float &v, float &rho, float &r) {
    const float x = pc[0], y = pc[1], z = pc[2];
    const float rho2 = x * x + z * z;
    rho = sqrtf(rho2);
    r = sqrtf(rho2 + y * y);
    const float Wf = (float)W;
    u = Kc[0] * atan2f(x, z) + Kc[2];
    u = u - Wf * floorf(u / Wf);
    if (u >= Wf) u = u - Wf;  // a tiny negative u rounds to W
    v = Kc[4] * atan2f(y, rho) + Kc[5];
    return r > near_plane && r < far_plane && rho > GSB_EQUIRECT_POLE_EPSILON * r;
}
// J = d(u, v)/d pc = diag(fx, fy) [z/rho^2 0 -x/rho^2; -x y/(r^2 rho) rho/r^2 -z y/(r^2 rho)], row-major 2x3: the Jacobian of
// Sigma' (pc detached, DESIGN section 3) and, with pc live, the position's
__device__ __forceinline__ void equirect_jacobian(float fx, float fy, const float *pc, float rho, float r, float *J) {
    const float x = pc[0], y = pc[1], z = pc[2];
    const float irho2 = 1.0f / (rho * rho), ir2 = 1.0f / (r * r);
    const float t = (y * ir2) / rho;
    J[0] = fx * (z * irho2); J[1] = 0.0f; J[2] = -(fx * (x * irho2));
    J[3] = -(fy * (x * t)); J[4] = fy * (rho * ir2); J[5] = -(fy * (z * t));
}
// The copy of a splat centre u nearest the tile column whose pixels start at tile_x0 (the blend kernels' WRAP staging)
__device__ __forceinline__ float equirect_wrap_u(float u, float tile_x0, float W) {
    return u + W * rintf(((tile_x0 + 0.5f * (float)GSB_TILE_WIDTH) - u) / W);
}
#endif

// ---- orthographic (parallel-projection) views (gsb200_forward_ortho / gsb200_backward_ortho; definition in include/gsb200.h).
// LENS_ORTHO is, like LENS_EQUIRECT, an internal model code of the per-point kernels' LENS switch, never a GsbLensArgs value.
// (u, v) = K[:2] (x, y, 1) and J = d(u, v)/d pc = K[:2,:2] [I 0] do not depend on z: the projection is linear.
constexpr int LENS_ORTHO = 0x4F52;

// Host, double: the r^2 bound of LensParams::r2_max (definition in include/gsb200.h), inf when the map never folds back.
// The smallest positive root of the derivative polynomial in t = r^2 (opencv) or t = theta^2 (fisheye) is bracketed
// between the roots of its derivative (recursively, degree <= 4) and bisected.
static inline double lens_poly(const double *c, int deg, double t) {
    double v = c[deg];
    for (int i = deg - 1; i >= 0; --i) v = v * t + c[i];
    return v;
}
// all roots of c[0] + c[1] t + ... + c[deg] t^deg in (lo, hi), ascending; returns their number
static inline int lens_poly_roots(const double *c, int deg, double lo, double hi, double *out) {
    while (deg > 0 && c[deg] == 0.0) --deg;
    if (deg == 0) return 0;
    double d[4], crit[4];
    for (int i = 1; i <= deg; ++i) d[i - 1] = i * c[i];
    const int nc = lens_poly_roots(d, deg - 1, lo, hi, crit);
    double edges[6];
    int ne = 0;
    edges[ne++] = lo;
    for (int i = 0; i < nc; ++i) edges[ne++] = crit[i];
    edges[ne++] = hi;
    int n = 0;
    for (int i = 0; i + 1 < ne; ++i) {
        double a = edges[i], b = edges[i + 1];
        double fa = lens_poly(c, deg, a), fb = lens_poly(c, deg, b);
        if (i > 0 && fa == 0.0) { out[n++] = a; continue; }  // a double root at a critical point
        if ((fa < 0.0) == (fb < 0.0) || fb == 0.0) continue;
        for (int it = 0; it < 200 && b - a > 0.0; ++it) {
            const double m = 0.5 * (a + b);
            if (m <= a || m >= b) break;
            const double fm = lens_poly(c, deg, m);
            if ((fm < 0.0) == (fa < 0.0)) { a = m; fa = fm; } else { b = m; }
        }
        out[n++] = 0.5 * (a + b);
    }
    return n;
}
static inline double lens_r2_bound(int model, const float *k) {
    const double inf = __builtin_inf();
    if (model == GSB_LENS_OPENCV) {
        const double c[4] = {1.0, 3.0 * k[0], 5.0 * k[1], 7.0 * k[4]};  // d(r rad)/dr in t = r^2
        double hi = 1.0;  // Cauchy bound of the positive roots
        for (int i = 3; i >= 1; --i)
            if (c[i] != 0.0) {
                double m = 0.0;
                for (int j = 0; j < i; ++j) m = fmax(m, fabs(c[j] / c[i]));
                hi = 2.0 * (1.0 + m);
                break;
            }
        double roots[4];
        return lens_poly_roots(c, 3, 0.0, hi, roots) > 0 ? roots[0] : inf;
    }
    if (model == GSB_LENS_FISHEYE) {
        const double half_pi = 1.5707963267948966;
        const double c[5] = {1.0, 3.0 * k[0], 5.0 * k[1], 7.0 * k[2], 9.0 * k[3]};  // d theta_d / d theta in t = theta^2
        double roots[4];
        double theta = half_pi;
        if (lens_poly_roots(c, 4, 0.0, half_pi * half_pi, roots) > 0) theta = fmin(theta, sqrt(roots[0]));
        if (theta >= half_pi) return inf;  // tan(pi/2): every point in front of the camera
        const double r = tan(theta);
        return r * r;
    }
    return inf;
}

// ---- mbarrier + TMA 1-D bulk copy (global -> shared), used by the radix sort (key tiles) and the per-point stage (feature rows)
#if defined(__CUDACC__) || defined(GSB_HOST_EMU)
#ifdef GSB_HOST_EMU  // tests/simt: host build under the SIMT emulator -- the bulk copy is a memcpy that has landed at once
__device__ __forceinline__ void mbar_init(unsigned long long *bar, unsigned int) { *bar = 0; }
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long *, unsigned int) {}
__device__ __forceinline__ void bulk_copy_g2s(void *dst_smem, const void *src_gmem, unsigned int bytes,
                                              unsigned long long *) {
    memcpy(dst_smem, src_gmem, bytes);
}
// every lane of the warp calls the wait (warp-uniform condition at both call sites): under the emulator it is a warp
// rendezvous, so the lane that issued the (immediate) copy has done so before any lane reads the destination
__device__ __forceinline__ void mbar_wait(unsigned long long *, unsigned int) { simt_emu::warp_exchange(0u); }
__device__ __forceinline__ void fence_proxy_async_smem() {}
#else
// ---- mbarrier / bulk-copy helpers (TMA 1-D bulk copy, global -> shared)
__device__ __forceinline__ unsigned int smem_addr(const void *p) {
    return (unsigned int)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(unsigned long long *bar, unsigned int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long *bar, unsigned int bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(void *dst_smem, const void *src_gmem, unsigned int bytes,
                                              unsigned long long *bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_addr(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_addr(bar))
        : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, unsigned int parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_addr(bar)),
        "r"(parity)
        : "memory");
}
// orders this CTA's earlier generic-proxy accesses to shared memory before a following bulk copy into the same bytes
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
#endif

#endif

// Work counters for the CPU-side emulation only (tests/simt, scripts/emu_work_stats.py); nothing in a device build.
#ifdef GSB_HOST_EMU
#define GSB_EMU_COUNT(slot, n) (simt_emu::counters()[slot] += (long long)(n))
#else
#define GSB_EMU_COUNT(slot, n) ((void)0)
#endif
enum EmuCounter {
    EC_BF_VISITS = 0,       // butterfly kernel: (warp, splat) visits
    EC_BF_VISITS_ANY = 1,   //   ... with at least one contributing pixel (these pay the butterfly + RED)
    EC_BF_PAIRS = 2,        //   contributing (pixel, splat) pairs
    EC_TB_SPLATS = 3,       // transposed kernel: (warp, splat) list entries
    EC_TB_CHUNKS = 4,       //   chunks processed
    EC_TB_ROWS = 5,         //   accumulator rows flushed (splats with a contributing pixel)
    EC_BATCHES = 6,         // staging batches (per CTA)
    EC_FW_VISITS = 7,       // forward blend: (warp, splat) visits
    EC_FW_PAIRS = 8,        //   (pixel, splat) pairs with alpha >= 1/255 on a live pixel (blended or saturating)
};

static inline int num_sms() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n <= 0) n = 132;
    }
    return n;
}

}  // namespace gsb
