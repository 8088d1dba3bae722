// robust_loss.cu -- per-pixel weights of the image loss (gsb200_train_step_robust, gsb200_robust_image_loss): a static
// per-view weight s (H,W) in [0,1] and / or the trimmed inlier mask of RobustNeRF (Sabour et al., CVPR 2023, section 4)
// computed from this iteration's residual.  For the image x (H,W,3) the image loss reads and its ground truth g (3,H,W):
//   c = clamp(x, 0, 1),  r = (|c0 - g0| + |c1 - g1| + |c2 - g2|) / 3,  bin = min(floor(r 4096), 4095)
//   b = the smallest bin with (float)cum(b) >= q (float)n over the n pixels with s > 0  (an exact integer histogram)
//   raw inlier: bin <= b;  3x3 inlier: (float)#raw inliers >= t3 (float)#neighbours, over the in-image 3x3 neighbours with s > 0
//   patch inlier: every pixel of a 16x16 tile when (float)#3x3 inliers >= t16 (float)#pixels, over the tile's pixels with s > 0
//   w = s [3x3 inlier or patch inlier]   (without the robust mask: w = s)
// The image loss (image_loss.cu, unchanged) then runs on the composite x' = w c + (1 - w) g, and its gradient is taken back
// to x as dL/dx = w 1[0 <= x <= 1] dL/dx'.  loss.py::robust_weight states the same in torch; it is this file's reference.
//   kernel 1 (robust only): per-CTA shared-memory histogram of the bins, added to a global one with integer atomics; the
//             last CTA (by ticket) scans it, writes b and clears the histogram for the next call;
//   kernel 2: one CTA per 16x16 tile with an 18x18 halo of raw inliers: the 3x3 rule, the tile count, w and x'; the two
//             counts of the stats it adds to are cleared right before it, so a call that stopped early leaves no trace;
//   kernel 3 (after the image loss wrote dL/dx'): dL/dx in place, and {inlier fraction, threshold}.
// Integer counts only: two calls are bit-identical.  Compiled with -fmad=false: the composite rounds like torch.
#include "common.cuh"

namespace gsb {

constexpr int RL_TILE = 16;
constexpr int RL_HALO = RL_TILE + 2;  // 18
constexpr int RL_THREADS = RL_TILE * RL_TILE;
constexpr int RL_WARPS = RL_THREADS / 32;
constexpr int RL_BINS = 4096;
constexpr int RL_BINS_PER_THREAD = RL_BINS / RL_THREADS;  // 16
constexpr int RL_HIST_MAX_BLOCKS = 512;
constexpr int RL_POST_MAX_BLOCKS = 1024;

struct RobustParams {
    const float *image_hwc;      // (H,W,3) x
    const float *gt_chw;         // (3,H,W) g
    const float *static_weight;  // (H,W) s, or null: 1 everywhere
    int H, W, tiles_x;
    int robust;
    float q, box_threshold, patch_threshold;
    float *weight_out;           // (H,W) w
    float *composite;            // (H,W,3) x'
    float *grad_hwc;             // post-pass: dL/dx' in, dL/dx out
    unsigned int *ticket;
    int *threshold_bin;          // b
    unsigned long long *counts;  // {n, pixels with s > 0 and w > 0}
    unsigned int *hist;          // [RL_BINS]
    float *stats_out;            // {inlier fraction, threshold}
};

__device__ __forceinline__ float rl_static(const RobustParams &p, long long i) {
    return p.static_weight ? __ldg(&p.static_weight[i]) : 1.0f;
}

__device__ __forceinline__ int rl_bin(const RobustParams &p, long long i) {
    const long long n = (long long)p.H * p.W;
    const float *x = p.image_hwc + 3 * i;
    const float r = (fabsf(fminf(fmaxf(__ldg(&x[0]), 0.0f), 1.0f) - __ldg(&p.gt_chw[i])) +
                     fabsf(fminf(fmaxf(__ldg(&x[1]), 0.0f), 1.0f) - __ldg(&p.gt_chw[n + i])) +
                     fabsf(fminf(fmaxf(__ldg(&x[2]), 0.0f), 1.0f) - __ldg(&p.gt_chw[2 * n + i]))) / 3.0f;
    return (int)fminf(floorf(r * (float)RL_BINS), (float)(RL_BINS - 1));
}

__global__ void __launch_bounds__(RL_THREADS) robust_hist_kernel(const RobustParams p) {
    __shared__ unsigned int s_hist[RL_BINS];
    __shared__ unsigned int s_tot[RL_THREADS];
    __shared__ bool s_last;
    const int tid = threadIdx.x;
    for (int k = tid; k < RL_BINS; k += RL_THREADS) s_hist[k] = 0u;
    __syncthreads();
    const long long n = (long long)p.H * p.W;
    // warp-uniform trip count; the lanes of a warp that share a bin add it once (a converged fit puts most residuals into
    // a few low bins, and same-address shared atomics serialise)
    const int lane = tid & 31;
    for (long long base = (long long)blockIdx.x * RL_THREADS + (tid - lane); base < n;
         base += (long long)gridDim.x * RL_THREADS) {
        const long long i = base + lane;
        const int bin = (i < n && rl_static(p, i) > 0.0f) ? rl_bin(p, i) : -1;
        const unsigned int peers = __match_any_sync(0xffffffffu, bin);
        if (bin >= 0 && lane == __ffs(peers) - 1) atomicAdd(&s_hist[bin], (unsigned int)__popc(peers));
    }
    __syncthreads();
    for (int k = tid; k < RL_BINS; k += RL_THREADS) {
        const unsigned int v = s_hist[k];
        if (v) atomicAdd(&p.hist[k], v);
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) s_last = atomicAdd(p.ticket, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!s_last) return;
    // the last CTA: every count is in.  Thread t owns bins [16 t, 16 t + 16); exactly one thread sees the predicate
    // (float)cum >= q (float)n turn true (it is monotone in the bin) and writes b
    __threadfence();
    unsigned int own[RL_BINS_PER_THREAD];
    unsigned int sum = 0u;
#pragma unroll
    for (int k = 0; k < RL_BINS_PER_THREAD; ++k) {
        own[k] = ((volatile unsigned int *)p.hist)[tid * RL_BINS_PER_THREAD + k];
        p.hist[tid * RL_BINS_PER_THREAD + k] = 0u;  // ready for the next call
        sum += own[k];
    }
    s_tot[tid] = sum;
    __syncthreads();
    unsigned long long before = 0ull, total = 0ull;
    for (int t = 0; t < RL_THREADS; ++t) {
        if (t < tid) before += s_tot[t];
        total += s_tot[t];
    }
    const float qn = p.q * (float)total;
    if (tid == 0 || !((float)before >= qn)) {
        unsigned long long cum = before;
        for (int k = 0; k < RL_BINS_PER_THREAD; ++k) {
            cum += own[k];
            if ((float)cum >= qn) {
                *p.threshold_bin = tid * RL_BINS_PER_THREAD + k;
                break;
            }
        }
    }
    if (tid == 0) *p.ticket = 0u;
}

__global__ void __launch_bounds__(RL_THREADS) robust_mask_kernel(const RobustParams p) {
    __shared__ unsigned char s_valid[RL_HALO][RL_HALO];
    __shared__ unsigned char s_raw[RL_HALO][RL_HALO];
    __shared__ unsigned int s_cnt[2][RL_WARPS];
    const int tid = threadIdx.x;
    const int r0 = (blockIdx.x / p.tiles_x) * RL_TILE, c0 = (blockIdx.x % p.tiles_x) * RL_TILE;
    if (p.robust) {
        const int b = *p.threshold_bin;
        for (int e = tid; e < RL_HALO * RL_HALO; e += RL_THREADS) {
            const int u = e / RL_HALO, v = e - u * RL_HALO;
            const int gr = r0 - 1 + u, gc = c0 - 1 + v;
            bool valid = false, raw = false;
            if (gr >= 0 && gr < p.H && gc >= 0 && gc < p.W) {
                const long long i = (long long)gr * p.W + gc;
                valid = rl_static(p, i) > 0.0f;
                raw = valid && rl_bin(p, i) <= b;
            }
            s_valid[u][v] = valid;
            s_raw[u][v] = raw;
        }
        __syncthreads();
    }
    const int li = tid / RL_TILE, lj = tid - li * RL_TILE;
    const long long i = (long long)(r0 + li) * p.W + (c0 + lj);
    const float s = rl_static(p, i);
    const bool valid = s > 0.0f;
    bool keep = true;
    if (p.robust) {
        int cnt = 0, inl = 0;
#pragma unroll
        for (int du = 0; du < 3; ++du) {
#pragma unroll
            for (int dv = 0; dv < 3; ++dv) {
                cnt += s_valid[li + du][lj + dv];
                inl += s_raw[li + du][lj + dv];
            }
        }
        const bool box = (float)inl >= p.box_threshold * (float)cnt;
        const unsigned int m = __ballot_sync(0xffffffffu, valid), k = __ballot_sync(0xffffffffu, valid && box);
        if ((tid & 31) == 0) {
            s_cnt[0][tid >> 5] = __popc(m);
            s_cnt[1][tid >> 5] = __popc(k);
        }
        __syncthreads();
        unsigned int tile_m = 0u, tile_k = 0u;
#pragma unroll
        for (int w = 0; w < RL_WARPS; ++w) {
            tile_m += s_cnt[0][w];
            tile_k += s_cnt[1][w];
        }
        keep = box || (float)tile_k >= p.patch_threshold * (float)tile_m;
        __syncthreads();  // s_cnt is reused below
    }
    const float w = s * (keep ? 1.0f : 0.0f);
    p.weight_out[i] = w;
    const long long n = (long long)p.H * p.W;
    const float rw = 1.0f - w;
    const float *x = p.image_hwc + 3 * i;
    float *xo = p.composite + 3 * i;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        const float c = fminf(fmaxf(__ldg(&x[ch]), 0.0f), 1.0f);
        xo[ch] = w * c + rw * __ldg(&p.gt_chw[ch * n + i]);
    }
    const unsigned int m = __ballot_sync(0xffffffffu, valid), k = __ballot_sync(0xffffffffu, valid && w > 0.0f);
    if ((tid & 31) == 0) {
        s_cnt[0][tid >> 5] = __popc(m);
        s_cnt[1][tid >> 5] = __popc(k);
    }
    __syncthreads();
    if (tid == 0) {
        unsigned long long tile_m = 0ull, tile_k = 0ull;
        for (int v = 0; v < RL_WARPS; ++v) {
            tile_m += s_cnt[0][v];
            tile_k += s_cnt[1][v];
        }
        if (tile_m) atomicAdd(&p.counts[0], tile_m);
        if (tile_k) atomicAdd(&p.counts[1], tile_k);
    }
}

__global__ void __launch_bounds__(RL_THREADS) robust_post_kernel(const RobustParams p) {
    const long long n = (long long)p.H * p.W;
    for (long long i = (long long)blockIdx.x * RL_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * RL_THREADS) {
        const float w = p.weight_out[i];
        const float *x = p.image_hwc + 3 * i;
        float *g = p.grad_hwc + 3 * i;
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
            const float xv = __ldg(&x[ch]);
            g[ch] = (xv >= 0.0f && xv <= 1.0f) ? w * g[ch] : 0.0f;  // torch.clamp hands the gradient through on [0, 1]
        }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        const unsigned long long valid = p.counts[0], kept = p.counts[1];
        p.stats_out[0] = valid ? (float)((double)kept / (double)valid) : 0.0f;
        p.stats_out[1] = p.robust ? (float)(*p.threshold_bin + 1) / (float)RL_BINS : 1.0f;
    }
}

// temp layout: [ticket: 16 B][b: 16 B][counts: 2 x 8 B, 32 B][histogram: 4096 x 4 B]; the ticket and the histogram are left
// zero by every call, the counts are cleared before the mask kernel
constexpr long long RL_OFF_BIN = 16, RL_OFF_COUNTS = 32, RL_OFF_HIST = 64;
constexpr long long RL_TEMP_BYTES = RL_OFF_HIST + 4LL * RL_BINS;

static inline int robust_hist_blocks(int H, int W) {
    const long long b = ((long long)H * W + 16LL * RL_THREADS - 1) / (16LL * RL_THREADS);
    return (int)(b < 1 ? 1 : (b > RL_HIST_MAX_BLOCKS ? RL_HIST_MAX_BLOCKS : b));
}

static inline int robust_post_blocks(int H, int W) {
    const long long b = ((long long)H * W + RL_THREADS - 1) / RL_THREADS;
    return (int)(b < 1 ? 1 : (b > RL_POST_MAX_BLOCKS ? RL_POST_MAX_BLOCKS : b));
}

static inline void robust_params(const float *image, const float *gt, const float *static_weight, int H, int W, int robust,
                                 float q, float box_threshold, float patch_threshold, float *weight_out, float *composite,
                                 float *grad, void *temp, float *stats_out, RobustParams *p) {
    char *base = static_cast<char *>(temp);
    p->image_hwc = image;
    p->gt_chw = gt;
    p->static_weight = static_weight;
    p->H = H;
    p->W = W;
    p->tiles_x = W / RL_TILE;
    p->robust = robust ? 1 : 0;
    p->q = q;
    p->box_threshold = box_threshold;
    p->patch_threshold = patch_threshold;
    p->weight_out = weight_out;
    p->composite = composite;
    p->grad_hwc = grad;
    p->ticket = reinterpret_cast<unsigned int *>(base);
    p->threshold_bin = reinterpret_cast<int *>(base + RL_OFF_BIN);
    p->counts = reinterpret_cast<unsigned long long *>(base + RL_OFF_COUNTS);
    p->hist = reinterpret_cast<unsigned int *>(base + RL_OFF_HIST);
    p->stats_out = stats_out;
}

#ifndef GSB_HOST_EMU
static inline void robust_params(const GsbRobustLossArgs &r, const float *image, const float *gt, int H, int W, float *grad,
                                 RobustParams *p) {
    robust_params(image, gt, r.static_weight, H, W, r.robust, r.inlier_quantile, r.box_threshold, r.patch_threshold,
                  r.weight_out, r.composite, grad, r.temp, r.stats_out2, p);
}

int launch_robust_pre(const GsbRobustLossArgs &r, const float *image, const float *gt, int H, int W, cudaStream_t stream) {
    RobustParams p;
    robust_params(r, image, gt, H, W, nullptr, &p);
    if (p.robust) {
        robust_hist_kernel<<<robust_hist_blocks(H, W), RL_THREADS, 0, stream>>>(p);
        GSB_CUDA_CHECK(cudaGetLastError());
    }
    GSB_CUDA_CHECK(cudaMemsetAsync(p.counts, 0, 2 * sizeof(unsigned long long), stream));
    robust_mask_kernel<<<(H / RL_TILE) * (W / RL_TILE), RL_THREADS, 0, stream>>>(p);
    GSB_CUDA_CHECK(cudaGetLastError());
    return GSB_OK;
}

int launch_robust_post(const GsbRobustLossArgs &r, const float *image, int H, int W, float *grad, cudaStream_t stream) {
    RobustParams p;
    robust_params(r, image, nullptr, H, W, grad, &p);
    robust_post_kernel<<<robust_post_blocks(H, W), RL_THREADS, 0, stream>>>(p);
    GSB_CUDA_CHECK(cudaGetLastError());
    return GSB_OK;
}
#endif

}  // namespace gsb

#ifndef GSB_HOST_EMU
extern "C" {

int64_t gsb200_robust_temp_bytes(int32_t camera_height, int32_t camera_width) {
    if (camera_height < gsb::RL_TILE || camera_width < gsb::RL_TILE || camera_height % gsb::RL_TILE ||
        camera_width % gsb::RL_TILE)
        return 0;
    return gsb::RL_TEMP_BYTES;
}

}  // extern "C"
#endif  // GSB_HOST_EMU
