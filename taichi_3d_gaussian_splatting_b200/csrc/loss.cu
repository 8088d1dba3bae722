// loss.cu -- fused clamp + L1 loss + its gradient (the step either side of the operator in the trainer:
// GaussianPointTrainer.py:168-175 clamps the rendered image to [0,1], LossFunction.py:29 takes
// mean |pred - gt|; autograd then runs ~8 elementwise kernels over the (H,W,3) image).  One pass here:
// 8 B read + 4 B written per element, deterministic two-level reduction (fixed grid, fixed order).
#include "common.cuh"

namespace gsb {

constexpr int L1_THREADS = 256;
constexpr int L1_MAX_BLOCKS = 1056;  // 132 SMs x 8

struct L1Params {
    const float *pred;
    const float *target;
    long long n;
    float grad_scale;  // upstream gradient / n
    int clamp01;
    float *grad;       // may be null
    float *partials;   // [L1_MAX_BLOCKS]
    unsigned int *ticket;
    float *loss;       // mean |clamp(pred) - target|
};

__global__ void __launch_bounds__(L1_THREADS) l1_loss_kernel(const L1Params p) {
    __shared__ double s_part[L1_THREADS / 32];
    __shared__ bool s_last;
    const long long n4 = p.n >> 2;
    const long long stride = (long long)gridDim.x * blockDim.x;
    const float4 *a4 = reinterpret_cast<const float4 *>(p.pred);
    const float4 *b4 = reinterpret_cast<const float4 *>(p.target);
    float4 *g4 = reinterpret_cast<float4 *>(p.grad);
    float acc = 0.0f;
    auto one = [&](float x, float y, float &g) {
        // torch.clamp passes the gradient where min <= x <= max; d|e|/de = sign(e) with sign(0) = 0
        const bool inside = !p.clamp01 || (x >= 0.0f && x <= 1.0f);
        const float xc = p.clamp01 ? fminf(fmaxf(x, 0.0f), 1.0f) : x;
        const float e = xc - y;
        acc += fabsf(e);
        g = inside ? (e > 0.0f ? p.grad_scale : (e < 0.0f ? -p.grad_scale : 0.0f)) : 0.0f;
    };
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        const float4 a = __ldg(a4 + i), b = __ldg(b4 + i);
        float4 g;
        one(a.x, b.x, g.x);
        one(a.y, b.y, g.y);
        one(a.z, b.z, g.z);
        one(a.w, b.w, g.w);
        if (g4) g4[i] = g;
    }
    if (blockIdx.x == 0 && threadIdx.x < (p.n & 3)) {  // tail (n not a multiple of 4)
        const long long i = (n4 << 2) + threadIdx.x;
        float g;
        one(p.pred[i], p.target[i], g);
        if (p.grad) p.grad[i] = g;
    }
    double d = (double)acc;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = d;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
#pragma unroll
        for (int w = 0; w < L1_THREADS / 32; ++w) t += s_part[w];
        p.partials[blockIdx.x] = (float)t;
        __threadfence();
        s_last = atomicAdd(p.ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (s_last && threadIdx.x < 32) {  // the last block to finish adds the partials in block order
        __threadfence();
        double t = 0.0;
        for (int b = threadIdx.x; b < (int)gridDim.x; b += 32) t += (double)((volatile float *)p.partials)[b];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        if (threadIdx.x == 0) {
            *p.loss = (float)(t / (double)p.n);
            *p.ticket = 0u;  // ready for the next call on this temp buffer
        }
    }
}

static inline L1Params l1_params(const float *pred, const float *target, long long n, int clamp01, float upstream,
                                 float *loss, float *grad, void *temp, long long *blocks_out) {
    L1Params p;
    p.pred = pred;
    p.target = target;
    p.n = n;
    p.grad_scale = upstream / (float)n;
    p.clamp01 = clamp01;
    p.grad = grad;
    p.ticket = reinterpret_cast<unsigned int *>(temp);
    p.partials = reinterpret_cast<float *>(temp) + 4;
    p.loss = loss;
    long long blocks = ((n >> 2) + L1_THREADS - 1) / L1_THREADS;
    if (blocks < 1) blocks = 1;
    if (blocks > L1_MAX_BLOCKS) blocks = L1_MAX_BLOCKS;
    *blocks_out = blocks;
    return p;
}

#ifndef GSB_HOST_EMU
int launch_l1_loss(const float *pred, const float *target, long long n, int clamp01, float upstream,
                   float *loss, float *grad, void *temp, cudaStream_t stream) {
    long long blocks = 1;
    const L1Params p = l1_params(pred, target, n, clamp01, upstream, loss, grad, temp, &blocks);
    l1_loss_kernel<<<(int)blocks, L1_THREADS, 0, stream>>>(p);
    GSB_CUDA_CHECK(cudaGetLastError());
    return GSB_OK;
}
#endif

}  // namespace gsb

#ifndef GSB_HOST_EMU
extern "C" {

int64_t gsb200_l1_loss_temp_bytes(void) { return (int64_t)(4 + gsb::L1_MAX_BLOCKS) * 4; }

int gsb200_l1_loss(const float *predicted_image, const float *ground_truth_image, int64_t num_elements,
                   int32_t clamp01, float upstream_grad, float *loss_out, float *grad_predicted_out, void *temp,
                   int64_t temp_bytes, void *stream) {
    using namespace gsb;
    if (num_elements <= 0 || !predicted_image || !ground_truth_image || !loss_out || !temp ||
        temp_bytes < gsb200_l1_loss_temp_bytes()) {
        set_error("l1_loss: bad arguments (n=%lld, temp_bytes=%lld)", (long long)num_elements, (long long)temp_bytes);
        return GSB_EINVAL;
    }
    if (reinterpret_cast<uintptr_t>(predicted_image) % 16 || reinterpret_cast<uintptr_t>(ground_truth_image) % 16 ||
        (grad_predicted_out && reinterpret_cast<uintptr_t>(grad_predicted_out) % 16) ||
        reinterpret_cast<uintptr_t>(temp) % 16) {
        set_error("l1_loss: image, gradient and temp pointers must be 16-byte aligned");
        return GSB_EINVAL;
    }
    return launch_l1_loss(predicted_image, ground_truth_image, num_elements, clamp01, upstream_grad, loss_out,
                          grad_predicted_out, temp, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
#endif  // GSB_HOST_EMU
