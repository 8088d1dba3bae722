// supervision_loss.cu -- the depth, mask and background terms of the fused train step (gsb200_train_step_aux), in two
// kernels around the unchanged image-loss kernels (image_loss.cu).  For one view, with I the rasterised image (H,W,3),
// S = pixel_accumulated_alpha, D = the rendered depth, optional targets d* (H,W), m (H,W) in [0,1] and bg (3 floats):
//   background:  I' = I + (1 - S) bg;  with a mask also gt' = gt m + (1 - m) bg (without one gt is already on bg)
//   image loss:  clamp + 0.8 L1 + 0.2 D-SSIM on (I', gt')                      (image_loss.cu, unchanged)
//   mask term:   w_m mean |S - m|
//   depth term:  w_d sum_valid |D - d*| / max(n_valid, 1), valid = d* finite and > 0 (0 / NaN = no measurement)
// loss.py::supervision_loss states the same loss in torch.
//   kernel 1 (pre-pass, per pixel): writes I' and gt' into the temp buffer, per-CTA partials of sum |S - m|,
//             sum_valid |D - d*| and n_valid; the last CTA adds them in a fixed order.
//   kernel 2 (post-pass, after the image loss wrote dL/dI' = dL/dI): dL/dS = w_m sign(S - m) / HW - sum_c dL/dI'_c bg_c,
//             dL/dD = valid ? w_d sign(D - d*) / n_valid : 0, and {total, mask term, depth term}.
// HBM-bound; fixed grid and summation order (two calls are bit-identical); each term's loads are skipped when it is off.
#include "common.cuh"

namespace gsb {

constexpr int SL_THREADS = 256;
constexpr int SL_WARPS = SL_THREADS / 32;
constexpr int SL_MAX_BLOCKS = 1024;  // per-CTA partials: at most 1024 per sum (the last CTA adds 4 per thread)

struct SupervisionParams {
    const float *image_hwc;     // (H,W,3) rasterised image
    const float *gt_chw;        // (3,H,W) ground truth
    const float *alpha;         // (H,W) S
    const float *depth;         // (H,W) D
    const float *depth_target;  // (H,W) or null: no depth term
    const float *mask_target;   // (H,W) or null
    const float *background;    // float[3] or null: no compositing
    int H, W;
    int mask_term;              // w_m > 0 (needs mask_target)
    float mask_weight;
    float mask_scale;           // w_m / (H W)
    float depth_weight;
    float *image_out;           // (H,W,3) I' (null without background)
    float *gt_out;              // (3,H,W) gt' (null without background + mask)
    const float *grad_image;    // (H,W,3) dL/dI' of the image loss (post-pass, background only)
    float *grad_alpha;          // (H,W) or null
    float *grad_depth;          // (H,W) or null
    double *partials;           // [3][SL_MAX_BLOCKS]: sum |S - m|, sum_valid |D - d*|, n_valid
    double *sums;               // [3] the same sums over the image
    unsigned int *ticket;
    const float *image_loss;    // {L, L1, 1 - SSIM} written by the image loss
    float *loss_out;            // {total, mask term, depth term}
};

// torch rounds every elementwise op of the composite on its own: no contraction into FMA here
#ifdef GSB_HOST_EMU
__device__ __forceinline__ float sl_mul(float a, float b) { return a * b; }
__device__ __forceinline__ float sl_add(float a, float b) { return a + b; }
#else
__device__ __forceinline__ float sl_mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float sl_add(float a, float b) { return __fadd_rn(a, b); }
#endif

__device__ __forceinline__ bool sl_valid_depth(float d) { return d > 0.0f && d <= 3.402823466e38f; }  // false for NaN, inf

// fixed-order sum of three values over the CTA (warp butterflies, then the warp totals in order); every thread gets them
__device__ __forceinline__ void sl_block_sum3(double v[3], double (*s_part)[SL_WARPS]) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    }
    __syncthreads();  // s_part may still be read by an earlier call
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int k = 0; k < 3; ++k) s_part[k][threadIdx.x >> 5] = v[k];
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        double t = 0.0;
#pragma unroll
        for (int w = 0; w < SL_WARPS; ++w) t += s_part[k][w];
        v[k] = t;
    }
}

__global__ void __launch_bounds__(SL_THREADS) supervision_pre_kernel(const SupervisionParams p) {
    __shared__ double s_part[3][SL_WARPS];
    __shared__ bool s_last;
    const int tid = threadIdx.x;
    const long long n = (long long)p.H * p.W;
    float bg0 = 0.0f, bg1 = 0.0f, bg2 = 0.0f;
    if (p.background) {
        bg0 = __ldg(&p.background[0]);
        bg1 = __ldg(&p.background[1]);
        bg2 = __ldg(&p.background[2]);
    }
    double v[3] = {0.0, 0.0, 0.0};
    for (long long i = (long long)blockIdx.x * SL_THREADS + tid; i < n; i += (long long)gridDim.x * SL_THREADS) {
        const float m = p.mask_target ? __ldg(&p.mask_target[i]) : 0.0f;
        if (p.image_out) {
            const float s = __ldg(&p.alpha[i]), r = 1.0f - s;
            const float *src = p.image_hwc + 3 * i;
            float *dst = p.image_out + 3 * i;
            dst[0] = sl_add(__ldg(&src[0]), sl_mul(r, bg0));
            dst[1] = sl_add(__ldg(&src[1]), sl_mul(r, bg1));
            dst[2] = sl_add(__ldg(&src[2]), sl_mul(r, bg2));
            if (p.gt_out) {
                const float rm = 1.0f - m;
                p.gt_out[i] = sl_add(sl_mul(__ldg(&p.gt_chw[i]), m), sl_mul(rm, bg0));
                p.gt_out[n + i] = sl_add(sl_mul(__ldg(&p.gt_chw[n + i]), m), sl_mul(rm, bg1));
                p.gt_out[2 * n + i] = sl_add(sl_mul(__ldg(&p.gt_chw[2 * n + i]), m), sl_mul(rm, bg2));
            }
        }
        if (p.mask_term) v[0] += (double)fabsf(__ldg(&p.alpha[i]) - m);
        if (p.depth_target) {
            const float d = __ldg(&p.depth_target[i]);
            if (sl_valid_depth(d)) {
                v[1] += (double)fabsf(__ldg(&p.depth[i]) - d);
                v[2] += 1.0;
            }
        }
    }
    sl_block_sum3(v, s_part);
    if (tid == 0) {
#pragma unroll
        for (int k = 0; k < 3; ++k) p.partials[k * SL_MAX_BLOCKS + blockIdx.x] = v[k];
        __threadfence();
        s_last = atomicAdd(p.ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last) return;
    // the last CTA to finish: every partial is written.  Thread t adds blocks t, t + 256, ... in order, then the CTA sum
    __threadfence();
    double w[3] = {0.0, 0.0, 0.0};
    for (int b = tid; b < (int)gridDim.x; b += SL_THREADS) {
#pragma unroll
        for (int k = 0; k < 3; ++k) w[k] += ((volatile double *)p.partials)[k * SL_MAX_BLOCKS + b];
    }
    sl_block_sum3(w, s_part);
    if (tid == 0) {
        p.sums[0] = w[0];
        p.sums[1] = w[1];
        p.sums[2] = w[2];
        *p.ticket = 0u;  // ready for the next call on this temp buffer
    }
}

__global__ void __launch_bounds__(SL_THREADS) supervision_post_kernel(const SupervisionParams p) {
    const long long n = (long long)p.H * p.W;
    const double n_valid = p.depth_target ? p.sums[2] : 0.0;
    const float depth_scale = p.depth_target ? p.depth_weight / (float)fmax(n_valid, 1.0) : 0.0f;
    float bg0 = 0.0f, bg1 = 0.0f, bg2 = 0.0f;
    if (p.background) {
        bg0 = __ldg(&p.background[0]);
        bg1 = __ldg(&p.background[1]);
        bg2 = __ldg(&p.background[2]);
    }
    for (long long i = (long long)blockIdx.x * SL_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * SL_THREADS) {
        if (p.grad_alpha) {
            float ga = 0.0f;
            if (p.mask_term) {
                const float e = __ldg(&p.alpha[i]) - __ldg(&p.mask_target[i]);
                ga = e > 0.0f ? p.mask_scale : (e < 0.0f ? -p.mask_scale : 0.0f);
            }
            if (p.background) {
                const float *g = p.grad_image + 3 * i;
                ga -= __ldg(&g[0]) * bg0 + __ldg(&g[1]) * bg1 + __ldg(&g[2]) * bg2;
            }
            p.grad_alpha[i] = ga;
        }
        if (p.depth_target) {
            const float d = __ldg(&p.depth_target[i]);
            float gd = 0.0f;
            if (sl_valid_depth(d)) {
                const float e = __ldg(&p.depth[i]) - d;
                gd = e > 0.0f ? depth_scale : (e < 0.0f ? -depth_scale : 0.0f);
            }
            p.grad_depth[i] = gd;
        }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        const double mask_loss = p.mask_term ? (double)p.mask_weight * p.sums[0] / (double)n : 0.0;
        const double depth_loss = p.depth_target ? (double)p.depth_weight * p.sums[1] / fmax(n_valid, 1.0) : 0.0;
        p.loss_out[0] = (float)((double)p.image_loss[0] + mask_loss + depth_loss);
        p.loss_out[1] = (float)mask_loss;
        p.loss_out[2] = (float)depth_loss;
    }
}

// temp layout: [ticket: 16 B][sums: 3 doubles][partials: 3 x SL_MAX_BLOCKS doubles][I' (H,W,3)][gt' (3,H,W)]
struct SupervisionLayout {
    long long off_sums, off_partials, off_image, off_gt, total;
};
static inline SupervisionLayout supervision_layout(int H, int W) {
    SupervisionLayout L;
    const long long n = (long long)H * W;
    L.off_sums = 16;
    L.off_partials = 64;
    L.off_image = (L.off_partials + 8LL * 3 * SL_MAX_BLOCKS + 255) / 256 * 256;
    L.off_gt = (L.off_image + 12 * n + 255) / 256 * 256;
    L.total = L.off_gt + 12 * n;
    return L;
}

static inline int supervision_blocks(int H, int W) {
    const long long b = ((long long)H * W + SL_THREADS - 1) / SL_THREADS;
    return (int)(b < 1 ? 1 : (b > SL_MAX_BLOCKS ? SL_MAX_BLOCKS : b));
}

// Fills the parameters of both kernels.  The terms that are off have null pointers; image_out / gt_out tell the caller
// which image and ground truth the image loss has to read.
static inline void supervision_params(const float *image, const float *gt, const float *alpha, const float *depth,
                                      const float *depth_target, const float *mask_target, const float *background,
                                      int H, int W, float depth_weight, float mask_weight, const float *grad_image,
                                      float *grad_alpha, float *grad_depth, const float *image_loss, float *loss_out,
                                      void *temp, SupervisionParams *p) {
    const SupervisionLayout L = supervision_layout(H, W);
    char *base = static_cast<char *>(temp);
    const bool depth_on = depth_weight > 0.0f && depth_target;
    const bool mask_on = mask_weight > 0.0f && mask_target;
    p->image_hwc = image;
    p->gt_chw = gt;
    p->alpha = alpha;
    p->depth = depth;
    p->depth_target = depth_on ? depth_target : nullptr;
    p->mask_target = (mask_on || background) ? mask_target : nullptr;
    p->background = background;
    p->H = H;
    p->W = W;
    p->mask_term = mask_on ? 1 : 0;
    p->mask_weight = mask_on ? mask_weight : 0.0f;
    p->mask_scale = mask_on ? mask_weight / (float)((long long)H * W) : 0.0f;
    p->depth_weight = depth_on ? depth_weight : 0.0f;
    p->image_out = background ? reinterpret_cast<float *>(base + L.off_image) : nullptr;
    p->gt_out = background && mask_target ? reinterpret_cast<float *>(base + L.off_gt) : nullptr;
    p->grad_image = grad_image;
    p->grad_alpha = (mask_on || background) ? grad_alpha : nullptr;
    p->grad_depth = depth_on ? grad_depth : nullptr;
    p->partials = reinterpret_cast<double *>(base + L.off_partials);
    p->sums = reinterpret_cast<double *>(base + L.off_sums);
    p->ticket = reinterpret_cast<unsigned int *>(base);
    p->image_loss = image_loss;
    p->loss_out = loss_out;
}

#ifndef GSB_HOST_EMU
static inline void supervision_params(const GsbSupervisionArgs &s, const float *image, const float *gt, const float *alpha,
                                      const float *depth, int H, int W, const float *grad_image, const float *image_loss,
                                      SupervisionParams *p) {
    supervision_params(image, gt, alpha, depth, s.depth_target, s.mask_target, s.background, H, W, s.depth_weight,
                       s.mask_weight, grad_image, s.grad_pixel_accumulated_alpha, s.grad_depth, image_loss, s.loss_out3,
                       s.temp, p);
}

int launch_supervision_pre(const GsbSupervisionArgs &s, const float *image, const float *gt, const float *alpha,
                           const float *depth, int H, int W, cudaStream_t stream, const float **loss_image,
                           const float **loss_gt) {
    SupervisionParams p;
    supervision_params(s, image, gt, alpha, depth, H, W, nullptr, nullptr, &p);
    *loss_image = p.image_out ? p.image_out : image;
    *loss_gt = p.gt_out ? p.gt_out : gt;
    supervision_pre_kernel<<<supervision_blocks(H, W), SL_THREADS, 0, stream>>>(p);
    GSB_CUDA_CHECK(cudaGetLastError());
    return GSB_OK;
}

int launch_supervision_post(const GsbSupervisionArgs &s, const float *image, const float *gt, const float *alpha,
                            const float *depth, int H, int W, const float *grad_image, const float *image_loss,
                            cudaStream_t stream) {
    SupervisionParams p;
    supervision_params(s, image, gt, alpha, depth, H, W, grad_image, image_loss, &p);
    supervision_post_kernel<<<supervision_blocks(H, W), SL_THREADS, 0, stream>>>(p);
    GSB_CUDA_CHECK(cudaGetLastError());
    return GSB_OK;
}
#endif

}  // namespace gsb

#ifndef GSB_HOST_EMU
extern "C" {

int64_t gsb200_supervision_temp_bytes(int32_t camera_height, int32_t camera_width) {
    if (camera_height <= 0 || camera_width <= 0) return 0;
    return gsb::supervision_layout(camera_height, camera_width).total;
}

}  // extern "C"
#endif  // GSB_HOST_EMU
