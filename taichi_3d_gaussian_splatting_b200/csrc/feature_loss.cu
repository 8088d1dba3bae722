// feature_loss.cu -- the feature term of the fused train step (gsb200_train_step_ext): a loss on the rendered per-Gaussian
// feature map F (H,W,C) of gsb200_forward_ext and its gradient dL/dF, the input of gsb200_backward_ext.  Two kinds:
//   cross entropy (semantic labels l (H,W) int32, labelled where 0 <= l < C):
//     w sum_labelled CE(softmax(F_p), l_p) / max(n_labelled, 1),  CE = log sum_c exp(F_pc - m_p) + m_p - F_pl, m_p = max_c F_pc
//     dL/dF_pc = w (softmax_c(F_p) - [c == l_p]) / max(n_labelled, 1)
//   l2 (distilled feature maps T (H,W,C), supervised where all C values are finite):
//     w sum_supervised sum_c (F_pc - T_pc)^2 / max(n_supervised C, 1),  dL/dF_pc = 2 w (F_pc - T_pc) / max(n_supervised C, 1)
// An unsupervised pixel gets a zero gradient.  loss.py::feature_loss states the same loss in torch.
//   kernel 1 (per pixel): per-CTA partials of the per-pixel terms and of the supervised-pixel count (double); the last CTA
//             adds them in a fixed order.
//   kernel 2 (per pixel): dL/dF and {feature term, n_supervised}.
// HBM-bound; fixed grid and summation order (two calls are bit-identical).  The C channels of a pixel live in registers:
// the kernels are instantiated for CP = 4, 8, 16 (the runtime C padded up) and read / write only the C real channels.
#include "common.cuh"

namespace gsb {

constexpr int FL_THREADS = 256;
constexpr int FL_WARPS = FL_THREADS / 32;
constexpr int FL_MAX_BLOCKS = 1024;  // per-CTA partials: at most 1024 per sum

struct FeatureLossParams {
    const float *fmap;       // (H,W,C) rendered feature map
    const int *labels;       // (H,W) cross entropy, else null
    const float *target;     // (H,W,C) l2, else null
    long long n;             // H W
    int C;
    float weight;
    float *grad;             // (H,W,C) dL/dF (pass 2)
    double *partials;        // [2][FL_MAX_BLOCKS]: sum of the per-pixel terms, n_supervised
    double *sums;            // [2] the same sums over the image
    unsigned int *ticket;
    float *loss_out;         // {feature term, n_supervised}
};

__device__ __forceinline__ bool fl_finite(float x) { return fabsf(x) <= 3.402823466e38f; }  // false for NaN, inf

// fixed-order sum of two values over the CTA (warp butterflies, then the warp totals in order); every thread gets them
__device__ __forceinline__ void fl_block_sum2(double v[2], double (*s_part)[FL_WARPS]) {
#pragma unroll
    for (int k = 0; k < 2; ++k) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    }
    __syncthreads();  // s_part may still be read by an earlier call
    if ((threadIdx.x & 31) == 0) {
        s_part[0][threadIdx.x >> 5] = v[0];
        s_part[1][threadIdx.x >> 5] = v[1];
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        double t = 0.0;
#pragma unroll
        for (int w = 0; w < FL_WARPS; ++w) t += s_part[k][w];
        v[k] = t;
    }
}

// The C channels of pixel i (padding: -inf for logits, so that they add nothing to the softmax; 0 otherwise).
template <int CP>
__device__ __forceinline__ void fl_load(const float *row, int C, float pad, float (&x)[CP]) {
#pragma unroll
    for (int c = 0; c < CP; ++c) x[c] = c < C ? __ldg(&row[c]) : pad;
}

// Cross entropy of one labelled pixel: returns log sum exp(x - m) + m - x_l; x is left as exp(x - m), s as their sum.
template <int CP>
__device__ __forceinline__ float fl_cross_entropy(float (&x)[CP], int label, float &s) {
    float m = x[0], xl = x[0];
#pragma unroll
    for (int c = 1; c < CP; ++c) {
        m = fmaxf(m, x[c]);
        if (c == label) xl = x[c];
    }
    s = 0.0f;
#pragma unroll
    for (int c = 0; c < CP; ++c) {
        x[c] = expf(x[c] - m);  // padding: exp(-inf) = 0
        s += x[c];
    }
    return logf(s) + (m - xl);
}

template <int CP>
__global__ void __launch_bounds__(FL_THREADS) feature_loss_sum_kernel(const FeatureLossParams p) {
    __shared__ double s_part[2][FL_WARPS];
    __shared__ bool s_last;
    const int tid = threadIdx.x;
    const int C = p.C;
    double v[2] = {0.0, 0.0};
    for (long long i = (long long)blockIdx.x * FL_THREADS + tid; i < p.n; i += (long long)gridDim.x * FL_THREADS) {
        float x[CP];
        if (p.labels) {
            const int l = __ldg(&p.labels[i]);
            if (l >= 0 && l < C) {
                fl_load<CP>(p.fmap + i * C, C, -INFINITY, x);
                float s;
                v[0] += (double)fl_cross_entropy<CP>(x, l, s);
                v[1] += 1.0;
            }
        } else {
            float t[CP];
            fl_load<CP>(p.target + i * C, C, 0.0f, t);
            bool ok = true;
#pragma unroll
            for (int c = 0; c < CP; ++c) ok = ok && fl_finite(t[c]);
            if (ok) {
                fl_load<CP>(p.fmap + i * C, C, 0.0f, x);
                float e = 0.0f;
#pragma unroll
                for (int c = 0; c < CP; ++c) {
                    const float d = x[c] - t[c];
                    e += d * d;
                }
                v[0] += (double)e;
                v[1] += 1.0;
            }
        }
    }
    fl_block_sum2(v, s_part);
    if (tid == 0) {
        p.partials[blockIdx.x] = v[0];
        p.partials[FL_MAX_BLOCKS + blockIdx.x] = v[1];
        __threadfence();
        s_last = atomicAdd(p.ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last) return;
    // the last CTA to finish: every partial is written.  Thread t adds blocks t, t + 256, ... in order, then the CTA sum
    __threadfence();
    double w[2] = {0.0, 0.0};
    for (int b = tid; b < (int)gridDim.x; b += FL_THREADS) {
        w[0] += ((volatile double *)p.partials)[b];
        w[1] += ((volatile double *)p.partials)[FL_MAX_BLOCKS + b];
    }
    fl_block_sum2(w, s_part);
    if (tid == 0) {
        p.sums[0] = w[0];
        p.sums[1] = w[1];
        *p.ticket = 0u;  // ready for the next call on this temp buffer
    }
}

template <int CP>
__global__ void __launch_bounds__(FL_THREADS) feature_loss_grad_kernel(const FeatureLossParams p) {
    const int C = p.C;
    const double n_sup = p.sums[1];
    const double denom = fmax(p.labels ? n_sup : n_sup * (double)C, 1.0);
    const float scale = (float)((p.labels ? 1.0 : 2.0) * (double)p.weight / denom);
    for (long long i = (long long)blockIdx.x * FL_THREADS + threadIdx.x; i < p.n; i += (long long)gridDim.x * FL_THREADS) {
        float x[CP];
        float *g = p.grad + i * C;
        if (p.labels) {
            const int l = __ldg(&p.labels[i]);
            if (l >= 0 && l < C) {
                fl_load<CP>(p.fmap + i * C, C, -INFINITY, x);
                float s;
                fl_cross_entropy<CP>(x, l, s);
                const float r = 1.0f / s;
#pragma unroll
                for (int c = 0; c < CP; ++c)
                    if (c < C) g[c] = scale * (x[c] * r - (c == l ? 1.0f : 0.0f));
            } else {
#pragma unroll
                for (int c = 0; c < CP; ++c)
                    if (c < C) g[c] = 0.0f;
            }
        } else {
            float t[CP];
            fl_load<CP>(p.target + i * C, C, 0.0f, t);
            bool ok = true;
#pragma unroll
            for (int c = 0; c < CP; ++c) ok = ok && fl_finite(t[c]);
            fl_load<CP>(p.fmap + i * C, C, 0.0f, x);
#pragma unroll
            for (int c = 0; c < CP; ++c)
                if (c < C) g[c] = ok ? scale * (x[c] - t[c]) : 0.0f;
        }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        p.loss_out[0] = (float)((double)p.weight * p.sums[0] / denom);
        p.loss_out[1] = (float)n_sup;
    }
}

// temp layout: [ticket: 16 B][sums: 2 doubles][partials: 2 x FL_MAX_BLOCKS doubles]
struct FeatureLossLayout {
    long long off_sums, off_partials, total;
};
static inline FeatureLossLayout feature_loss_layout() {
    FeatureLossLayout L;
    L.off_sums = 16;
    L.off_partials = 64;
    L.total = L.off_partials + 8LL * 2 * FL_MAX_BLOCKS;
    return L;
}

static inline int feature_loss_blocks(int H, int W) {
    const long long b = ((long long)H * W + FL_THREADS - 1) / FL_THREADS;
    return (int)(b < 1 ? 1 : (b > FL_MAX_BLOCKS ? FL_MAX_BLOCKS : b));
}

// The compile-time channel width of a runtime C in 1..16.
static inline int feature_loss_width(int C) { return C <= 4 ? 4 : (C <= 8 ? 8 : 16); }

// labels: cross entropy; else target: l2.
static inline void feature_loss_params(const float *fmap, const int *labels, const float *target, int H, int W, int C,
                                       float weight, float *grad, float *loss_out, void *temp, FeatureLossParams *p) {
    const FeatureLossLayout L = feature_loss_layout();
    char *base = static_cast<char *>(temp);
    p->fmap = fmap;
    p->labels = labels;
    p->target = labels ? nullptr : target;
    p->n = (long long)H * W;
    p->C = C;
    p->weight = weight;
    p->grad = grad;
    p->partials = reinterpret_cast<double *>(base + L.off_partials);
    p->sums = reinterpret_cast<double *>(base + L.off_sums);
    p->ticket = reinterpret_cast<unsigned int *>(base);
    p->loss_out = loss_out;
}

#ifndef GSB_HOST_EMU
template <int CP>
static int launch_feature_loss_cp(const FeatureLossParams &p, int blocks, cudaStream_t stream) {
    feature_loss_sum_kernel<CP><<<blocks, FL_THREADS, 0, stream>>>(p);
    GSB_CUDA_CHECK(cudaGetLastError());
    feature_loss_grad_kernel<CP><<<blocks, FL_THREADS, 0, stream>>>(p);
    GSB_CUDA_CHECK(cudaGetLastError());
    return GSB_OK;
}

int launch_feature_loss(const GsbFeatureTrainArgs &x, int H, int W, cudaStream_t stream) {
    const GsbExtraFeatureArgs &e = x.features;
    FeatureLossParams p;
    feature_loss_params(e.rasterized, x.loss_kind == GSB_FEATURE_LOSS_CROSS_ENTROPY ? x.labels : nullptr, x.target, H, W,
                        e.channels, x.weight, const_cast<float *>(e.grad_rasterized), x.loss_out2, x.temp, &p);
    const int blocks = feature_loss_blocks(H, W);
    switch (feature_loss_width(e.channels)) {
        case 4: return launch_feature_loss_cp<4>(p, blocks, stream);
        case 8: return launch_feature_loss_cp<8>(p, blocks, stream);
        default: return launch_feature_loss_cp<16>(p, blocks, stream);
    }
}
#endif

}  // namespace gsb

#ifndef GSB_HOST_EMU
extern "C" {

int64_t gsb200_feature_loss_temp_bytes(int32_t camera_height, int32_t camera_width) {
    if (camera_height <= 0 || camera_width <= 0) return 0;
    return gsb::feature_loss_layout().total;
}

}  // extern "C"
#endif  // GSB_HOST_EMU
