// mcmc.cu -- MCMC densification (Kheradmand et al., "3D Gaussian Splatting as Markov Chain Monte Carlo", NeurIPS 2024;
// the definition is in include/gsb200.h): four kernels.
//   mcmc_regulariser_kernel       every iteration, between the backward and Adam: adds the gradient of the opacity and scale
//                                 L1 terms into columns 4..7 of the dense (N,56) gradient and sums the two terms in double
//                                 (per-CTA partials, the last CTA adds them in a fixed order).  36 B read + 16 B written per
//                                 valid row.
//   mcmc_noise_kernel             every iteration, after Adam: xyz += Sigma eps noise_scale g(o), eps from Philox4x32-10 with
//                                 counter (row, step).  45 B read + 12 B written per valid row.
//   mcmc_relocate_sources_kernel  at a refinement, one thread per drawn source: new logit and log-scales (double), moments 0.
//   mcmc_relocate_copy_kernel     then one warp per destination row: the source's updated row copied, mask cleared, moments 0.
// mcmc.py states the same arithmetic in torch.
#include "common.cuh"

namespace gsb {

constexpr int MC_THREADS = 256;
constexpr int MC_WARPS = MC_THREADS / 32;
constexpr int MC_MAX_BLOCKS = 1024;  // per-CTA partials: at most 1024 per sum (the last CTA adds 4 per thread)
constexpr int MC_ROW4 = GSB_FEATURE_DIM / 4;  // float4 per feature row
static_assert(GSB_FEATURE_DIM == 56, "the feature row is 14 float4");

__device__ __forceinline__ float mc_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

// ------------------------------------------------------------------------------------------------ regulariser
struct McmcRegulariserParams {
    const float4 *features;     // (N,14) float4
    const signed char *invalid_mask;
    float4 *grad_features;      // (N,14) float4
    long long N;
    float grad_opacity;         // lambda_o / n_v
    float grad_scale;           // lambda_s / (3 n_v)
    double term_opacity;        // the same in double, for the terms
    double term_scale;
    double *partials;           // [2][MC_MAX_BLOCKS]
    unsigned int *ticket;
    float *terms_out;           // {opacity term, scale term}
    const long long *skip_flag; // optional device flag: non-zero = no-op
};

// fixed-order sum of two values over the CTA (warp butterflies, then the warp totals in order); every thread gets them
__device__ __forceinline__ void mc_block_sum2(double v[2], double (*s_part)[MC_WARPS]) {
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
        for (int w = 0; w < MC_WARPS; ++w) t += s_part[k][w];
        v[k] = t;
    }
}

__global__ void __launch_bounds__(MC_THREADS) mcmc_regulariser_kernel(const McmcRegulariserParams p) {
    __shared__ double s_part[2][MC_WARPS];
    __shared__ bool s_last;
    if (p.skip_flag != nullptr && *p.skip_flag != 0) return;
    const int tid = threadIdx.x;
    double v[2] = {0.0, 0.0};
    for (long long i = (long long)blockIdx.x * MC_THREADS + tid; i < p.N; i += (long long)gridDim.x * MC_THREADS) {
        if (p.invalid_mask[i] != 0) continue;
        const float4 f = __ldg(p.features + i * MC_ROW4 + 1);  // s0 s1 s2 logit
        const float o = mc_sigmoid(f.w);
        const float e0 = expf(f.x), e1 = expf(f.y), e2 = expf(f.z);
        float4 g = p.grad_features[i * MC_ROW4 + 1];
        g.x += p.grad_scale * e0;
        g.y += p.grad_scale * e1;
        g.z += p.grad_scale * e2;
        g.w += p.grad_opacity * (o * (1.0f - o));
        p.grad_features[i * MC_ROW4 + 1] = g;
        v[0] += (double)o;
        v[1] += (double)e0 + (double)e1 + (double)e2;
    }
    mc_block_sum2(v, s_part);
    if (tid == 0) {
        p.partials[blockIdx.x] = v[0];
        p.partials[MC_MAX_BLOCKS + blockIdx.x] = v[1];
        __threadfence();
        s_last = atomicAdd(p.ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last) return;
    // the last CTA to finish: every partial is written.  Thread t adds blocks t, t + 256, ... in order, then the CTA sum
    __threadfence();
    double w[2] = {0.0, 0.0};
    for (int b = tid; b < (int)gridDim.x; b += MC_THREADS) {
        w[0] += ((volatile double *)p.partials)[b];
        w[1] += ((volatile double *)p.partials)[MC_MAX_BLOCKS + b];
    }
    mc_block_sum2(w, s_part);
    if (tid == 0) {
        p.terms_out[0] = (float)(p.term_opacity * w[0]);
        p.terms_out[1] = (float)(p.term_scale * w[1]);
        *p.ticket = 0u;  // ready for the next call on this temp buffer
    }
}

// temp layout: [ticket: 16 B][partials: 2 x MC_MAX_BLOCKS doubles]
static inline long long mcmc_temp_bytes() { return 16 + 8LL * 2 * MC_MAX_BLOCKS; }

static inline int mcmc_regulariser_blocks(long long N) {
    const long long b = (N + MC_THREADS - 1) / MC_THREADS;
    return (int)(b < 1 ? 1 : (b > MC_MAX_BLOCKS ? MC_MAX_BLOCKS : b));
}

static inline McmcRegulariserParams mcmc_regulariser_params(const float *features, const signed char *invalid_mask,
                                                            float *grad_features, long long N, long long num_valid,
                                                            float lambda_opacity, float lambda_scale, float *terms_out,
                                                            void *temp) {
    McmcRegulariserParams p;
    const double n_v = num_valid > 0 ? (double)num_valid : 1.0;
    p.features = reinterpret_cast<const float4 *>(features);
    p.invalid_mask = invalid_mask;
    p.grad_features = reinterpret_cast<float4 *>(grad_features);
    p.N = N;
    p.term_opacity = (double)lambda_opacity / n_v;
    p.term_scale = (double)lambda_scale / (3.0 * n_v);
    p.grad_opacity = (float)p.term_opacity;
    p.grad_scale = (float)p.term_scale;
    p.ticket = reinterpret_cast<unsigned int *>(temp);
    p.partials = reinterpret_cast<double *>(static_cast<char *>(temp) + 16);
    p.terms_out = terms_out;
    p.skip_flag = nullptr;
    return p;
}

// ------------------------------------------------------------------------------------------------ noise
struct McmcNoiseParams {
    float *pointcloud;          // (N,3)
    const float4 *features;     // (N,14) float4
    const signed char *invalid_mask;
    long long N;
    float noise_scale, gate_k, min_opacity;
    unsigned int key0, key1;    // seed low / high
    unsigned int step0, step1;  // step low / high
    const long long *skip_flag; // optional device flag: non-zero = no-op
};

__device__ __forceinline__ void mc_mulhilo(unsigned int a, unsigned int b, unsigned int &hi, unsigned int &lo) {
    const unsigned long long prod = (unsigned long long)a * b;
    hi = (unsigned int)(prod >> 32);
    lo = (unsigned int)prod;
}

// Philox4x32-10: counter c[4], key (k0, k1); the result replaces c
__device__ __forceinline__ void mc_philox4x32_10(unsigned int c[4], unsigned int k0, unsigned int k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        unsigned int hi0, lo0, hi1, lo1;
        mc_mulhilo(0xD2511F53u, c[0], hi0, lo0);
        mc_mulhilo(0xCD9E8D57u, c[2], hi1, lo1);
        const unsigned int n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
        c[0] = n0;
        c[1] = lo1;
        c[2] = n2;
        c[3] = lo0;
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
}

// ((x >> 9) + 0.5) 2^-23: 24 significant bits, exact in float32, in (0, 1)
__device__ __forceinline__ float mc_uniform(unsigned int x) { return ((float)(x >> 9) + 0.5f) * 1.1920928955078125e-7f; }

// sin and cos of 2 pi u
__device__ __forceinline__ void mc_sincos_2pi(float u, float *s, float *c) {
#ifdef GSB_HOST_EMU
    const double a = 6.283185307179586476925 * (double)u;
    *s = (float)sin(a);
    *c = (float)cos(a);
#else
    sincospif(2.0f * u, s, c);
#endif
}

__global__ void __launch_bounds__(MC_THREADS) mcmc_noise_kernel(const McmcNoiseParams p) {
    if (p.skip_flag != nullptr && *p.skip_flag != 0) return;
    const long long i = (long long)blockIdx.x * MC_THREADS + threadIdx.x;
    if (i >= p.N || p.invalid_mask[i] != 0) return;
    const float4 q = __ldg(p.features + i * MC_ROW4);
    const float4 sl = __ldg(p.features + i * MC_ROW4 + 1);  // s0 s1 s2 logit
    const float o = mc_sigmoid(sl.w);
    // g(o) = 1 / (1 + exp(-k ((1 - o) - (1 - tau)))); exp overflows to inf for an opaque row: the gate is then exactly 0
    const float gate = 1.0f / (1.0f + expf(-p.gate_k * ((1.0f - o) - (1.0f - p.min_opacity))));
    const float amp = p.noise_scale * gate;

    unsigned int c[4] = {(unsigned int)((unsigned long long)i & 0xffffffffull), (unsigned int)((unsigned long long)i >> 32),
                         p.step0, p.step1};
    mc_philox4x32_10(c, p.key0, p.key1);
    const float r0 = sqrtf(-2.0f * logf(mc_uniform(c[0]))), r1 = sqrtf(-2.0f * logf(mc_uniform(c[2])));
    float sn0, cs0, sn1, cs1;
    mc_sincos_2pi(mc_uniform(c[1]), &sn0, &cs0);
    mc_sincos_2pi(mc_uniform(c[3]), &sn1, &cs1);
    const float e0 = r0 * cs0, e1 = r0 * sn0, e2 = r1 * cs1;
    (void)sn1;

    // R of the normalised quaternion (xyzw), utils.quaternion_to_rotation_matrix_torch
    const float inv = 1.0f / sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
    const float x = q.x * inv, y = q.y * inv, z = q.z * inv, w = q.w * inv;
    const float R00 = 1.0f - 2.0f * (y * y + z * z), R01 = 2.0f * (x * y - z * w), R02 = 2.0f * (x * z + y * w);
    const float R10 = 2.0f * (x * y + z * w), R11 = 1.0f - 2.0f * (x * x + z * z), R12 = 2.0f * (y * z - x * w);
    const float R20 = 2.0f * (x * z - y * w), R21 = 2.0f * (y * z + x * w), R22 = 1.0f - 2.0f * (x * x + y * y);
    // Sigma eps = R diag(exp(2 s)) (R^T eps)
    const float v0 = expf(2.0f * sl.x) * (R00 * e0 + R10 * e1 + R20 * e2);
    const float v1 = expf(2.0f * sl.y) * (R01 * e0 + R11 * e1 + R21 * e2);
    const float v2 = expf(2.0f * sl.z) * (R02 * e0 + R12 * e1 + R22 * e2);
    float *xyz = p.pointcloud + 3 * i;
    xyz[0] += amp * (R00 * v0 + R01 * v1 + R02 * v2);
    xyz[1] += amp * (R10 * v0 + R11 * v1 + R12 * v2);
    xyz[2] += amp * (R20 * v0 + R21 * v1 + R22 * v2);
}

static inline McmcNoiseParams mcmc_noise_params(float *pointcloud, const float *features, const signed char *invalid_mask,
                                                long long N, float noise_scale, float gate_k, float min_opacity,
                                                unsigned long long seed, long long step) {
    McmcNoiseParams p;
    p.pointcloud = pointcloud;
    p.features = reinterpret_cast<const float4 *>(features);
    p.invalid_mask = invalid_mask;
    p.N = N;
    p.noise_scale = noise_scale;
    p.gate_k = gate_k;
    p.min_opacity = min_opacity;
    p.key0 = (unsigned int)(seed & 0xffffffffull);
    p.key1 = (unsigned int)(seed >> 32);
    p.step0 = (unsigned int)((unsigned long long)step & 0xffffffffull);
    p.step1 = (unsigned int)((unsigned long long)step >> 32);
    p.skip_flag = nullptr;
    return p;
}

// ------------------------------------------------------------------------------------------------ relocation
// C(i, k) for i < GSB_MCMC_N_MAX, built at compile time (C(50, 25) ~ 1.3e14 is exact in double)
struct McmcBinomial {
    double c[GSB_MCMC_N_MAX][GSB_MCMC_N_MAX];
    constexpr McmcBinomial() : c() {
        for (int i = 0; i < GSB_MCMC_N_MAX; ++i) {
            for (int k = 0; k < GSB_MCMC_N_MAX; ++k) c[i][k] = 0.0;
            c[i][0] = 1.0;
            for (int k = 1; k <= i; ++k) c[i][k] = c[i - 1][k - 1] + (k <= i - 1 ? c[i - 1][k] : 0.0);
        }
    }
};
#ifdef GSB_HOST_EMU
static const McmcBinomial mc_binomial = McmcBinomial();
#else
__device__ const McmcBinomial mc_binomial = McmcBinomial();
#endif

struct McmcRelocateParams {
    long long N;
    long long num_sources;
    const int *source_ids, *source_counts;
    long long num_destinations;
    const int *destination_ids, *destination_sources;
    float *pointcloud;
    float4 *features;
    signed char *invalid_mask;
    int *object_id;
    float *extra_features;
    int channels;
    double min_opacity;
    float4 *feature_exp_avg, *feature_exp_avg_sq;
    float *position_exp_avg, *position_exp_avg_sq;
    float *extra_exp_avg, *extra_exp_avg_sq;
};

__global__ void __launch_bounds__(MC_THREADS) mcmc_relocate_sources_kernel(const McmcRelocateParams p) {
    const long long j = (long long)blockIdx.x * MC_THREADS + threadIdx.x;
    if (j >= p.num_sources) return;
    const long long id = p.source_ids[j];
    if (id < 0 || id >= p.N) return;
    long long n = (long long)p.source_counts[j] + 1;
    n = n < 1 ? 1 : (n > GSB_MCMC_N_MAX ? GSB_MCMC_N_MAX : n);
    float4 f = p.features[id * MC_ROW4 + 1];  // s0 s1 s2 logit
    const double o = 1.0 / (1.0 + exp(-(double)f.w));
    const double o_new = -expm1(log1p(-o) / (double)n);  // 1 - (1 - o)^(1/n)
    double D = 0.0;
    for (int i = 1; i <= (int)n; ++i) {
        double pw = o_new, sign = 1.0;  // o_new^(k+1), (-1)^k
        for (int k = 0; k < i; ++k) {
            D += mc_binomial.c[i - 1][k] * sign * pw / sqrt((double)(k + 1));
            pw *= o_new;
            sign = -sign;
        }
    }
    const float shift = (float)log(o / D);
    f.x += shift;
    f.y += shift;
    f.z += shift;
    const double oc = fmin(fmax(o_new, p.min_opacity), 1.0 - 1e-7);
    f.w = (float)log(oc / (1.0 - oc));
    p.features[id * MC_ROW4 + 1] = f;
    const float4 zero = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    if (p.feature_exp_avg) {
        for (int k = 0; k < MC_ROW4; ++k) {
            p.feature_exp_avg[id * MC_ROW4 + k] = zero;
            p.feature_exp_avg_sq[id * MC_ROW4 + k] = zero;
        }
    }
    if (p.position_exp_avg) {
        for (int k = 0; k < 3; ++k) {
            p.position_exp_avg[id * 3 + k] = 0.0f;
            p.position_exp_avg_sq[id * 3 + k] = 0.0f;
        }
    }
    if (p.extra_exp_avg) {
        for (int k = 0; k < p.channels; ++k) {
            p.extra_exp_avg[id * p.channels + k] = 0.0f;
            p.extra_exp_avg_sq[id * p.channels + k] = 0.0f;
        }
    }
}

// one warp per destination row; the sources kernel has finished (stream order)
__global__ void __launch_bounds__(MC_THREADS) mcmc_relocate_copy_kernel(const McmcRelocateParams p) {
    const long long d = (long long)blockIdx.x * MC_WARPS + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (d >= p.num_destinations) return;
    const long long dst = p.destination_ids[d], src = p.destination_sources[d];
    if (dst < 0 || dst >= p.N || src < 0 || src >= p.N) return;
    const float4 zero = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    if (lane < MC_ROW4) {
        p.features[dst * MC_ROW4 + lane] = p.features[src * MC_ROW4 + lane];
        if (p.feature_exp_avg) {
            p.feature_exp_avg[dst * MC_ROW4 + lane] = zero;
            p.feature_exp_avg_sq[dst * MC_ROW4 + lane] = zero;
        }
    }
    if (lane < 3) {
        p.pointcloud[dst * 3 + lane] = p.pointcloud[src * 3 + lane];
        if (p.position_exp_avg) {
            p.position_exp_avg[dst * 3 + lane] = 0.0f;
            p.position_exp_avg_sq[dst * 3 + lane] = 0.0f;
        }
    }
    if (lane < p.channels && p.extra_features) {
        p.extra_features[dst * p.channels + lane] = p.extra_features[src * p.channels + lane];
        if (p.extra_exp_avg) {
            p.extra_exp_avg[dst * p.channels + lane] = 0.0f;
            p.extra_exp_avg_sq[dst * p.channels + lane] = 0.0f;
        }
    }
    if (lane == 16) p.object_id[dst] = p.object_id[src];
    if (lane == 17) p.invalid_mask[dst] = 0;
}

static inline McmcRelocateParams mcmc_relocate_params(const GsbMcmcRelocateArgs &a) {
    McmcRelocateParams p;
    p.N = a.num_points;
    p.num_sources = a.num_sources;
    p.source_ids = a.source_ids;
    p.source_counts = a.source_counts;
    p.num_destinations = a.num_destinations;
    p.destination_ids = a.destination_ids;
    p.destination_sources = a.destination_sources;
    p.pointcloud = a.pointcloud;
    p.features = reinterpret_cast<float4 *>(a.pointcloud_features);
    p.invalid_mask = reinterpret_cast<signed char *>(a.point_invalid_mask);
    p.object_id = a.point_object_id;
    p.extra_features = a.extra_features;
    p.channels = a.extra_features ? a.channels : 0;
    p.min_opacity = (double)a.min_opacity;
    p.feature_exp_avg = reinterpret_cast<float4 *>(a.feature_exp_avg);
    p.feature_exp_avg_sq = reinterpret_cast<float4 *>(a.feature_exp_avg_sq);
    p.position_exp_avg = a.position_exp_avg;
    p.position_exp_avg_sq = a.position_exp_avg_sq;
    p.extra_exp_avg = a.extra_exp_avg;
    p.extra_exp_avg_sq = a.extra_exp_avg_sq;
    return p;
}

#ifndef GSB_HOST_EMU
int launch_mcmc_regulariser(const float *features, const int8_t *invalid_mask, float *grad_features, long long N,
                            long long num_valid, float lambda_opacity, float lambda_scale, float *terms_out, void *temp,
                            const long long *skip_flag, cudaStream_t stream) {
    McmcRegulariserParams p = mcmc_regulariser_params(features, reinterpret_cast<const signed char *>(invalid_mask),
                                                      grad_features, N, num_valid, lambda_opacity, lambda_scale, terms_out,
                                                      temp);
    p.skip_flag = skip_flag;
    mcmc_regulariser_kernel<<<mcmc_regulariser_blocks(N), MC_THREADS, 0, stream>>>(p);
    GSB_CUDA_CHECK(cudaGetLastError());
    return GSB_OK;
}

int launch_mcmc_noise(float *pointcloud, const float *features, const int8_t *invalid_mask, long long N, float noise_scale,
                      float gate_k, float min_opacity, unsigned long long seed, long long step, const long long *skip_flag,
                      cudaStream_t stream) {
    if (N <= 0) return GSB_OK;
    McmcNoiseParams p = mcmc_noise_params(pointcloud, features, reinterpret_cast<const signed char *>(invalid_mask), N,
                                          noise_scale, gate_k, min_opacity, seed, step);
    p.skip_flag = skip_flag;
    mcmc_noise_kernel<<<(unsigned int)((N + MC_THREADS - 1) / MC_THREADS), MC_THREADS, 0, stream>>>(p);
    GSB_CUDA_CHECK(cudaGetLastError());
    return GSB_OK;
}
#endif

}  // namespace gsb

#ifndef GSB_HOST_EMU
extern "C" {

int64_t gsb200_mcmc_temp_bytes(void) { return gsb::mcmc_temp_bytes(); }

int gsb200_mcmc_relocate(const GsbMcmcRelocateArgs *a) {
    using namespace gsb;
    auto misaligned16 = [](const void *p) { return reinterpret_cast<uintptr_t>(p) % 16 != 0; };
    if (!a || a->num_points < 0 || a->num_sources < 0 || a->num_sources > a->num_points || a->num_destinations < 0 ||
        a->num_destinations > a->num_points) {
        set_error("mcmc_relocate: NULL args, or a count outside [0, num_points]");
        return GSB_EINVAL;
    }
    if ((a->num_sources > 0 && (!a->source_ids || !a->source_counts)) ||
        (a->num_destinations > 0 && (!a->destination_ids || !a->destination_sources))) {
        set_error("mcmc_relocate: NULL id array with a non-zero count");
        return GSB_EINVAL;
    }
    if (!a->pointcloud || !a->pointcloud_features || !a->point_invalid_mask || !a->point_object_id ||
        misaligned16(a->pointcloud_features)) {
        set_error("mcmc_relocate: NULL scene tensor, or pointcloud_features not 16-byte aligned");
        return GSB_EINVAL;
    }
    if (a->extra_features && (a->channels < 1 || a->channels > 16)) {
        set_error("mcmc_relocate: channels must be in 1..16 (got %d)", a->channels);
        return GSB_EINVAL;
    }
    if (!a->feature_exp_avg != !a->feature_exp_avg_sq || !a->position_exp_avg != !a->position_exp_avg_sq ||
        !a->extra_exp_avg != !a->extra_exp_avg_sq || (a->extra_exp_avg && !a->extra_features) ||
        misaligned16(a->feature_exp_avg) || misaligned16(a->feature_exp_avg_sq)) {
        set_error("mcmc_relocate: a moment pair needs both halves (the feature moments 16-byte aligned), the extra moments "
                  "need extra_features");
        return GSB_EINVAL;
    }
    if (!(a->min_opacity > 0.0f && a->min_opacity < 1.0f)) {
        set_error("mcmc_relocate: min_opacity must be in (0, 1) (got %g)", (double)a->min_opacity);
        return GSB_EINVAL;
    }
    const McmcRelocateParams p = mcmc_relocate_params(*a);
    cudaStream_t st = static_cast<cudaStream_t>(a->stream);
    if (p.num_sources > 0) {
        mcmc_relocate_sources_kernel<<<(unsigned int)((p.num_sources + MC_THREADS - 1) / MC_THREADS), MC_THREADS, 0, st>>>(p);
        GSB_CUDA_CHECK(cudaGetLastError());
    }
    if (p.num_destinations > 0) {
        mcmc_relocate_copy_kernel<<<(unsigned int)((p.num_destinations + MC_WARPS - 1) / MC_WARPS), MC_THREADS, 0, st>>>(p);
        GSB_CUDA_CHECK(cudaGetLastError());
    }
    return GSB_OK;
}

}  // extern "C"
#endif  // GSB_HOST_EMU
