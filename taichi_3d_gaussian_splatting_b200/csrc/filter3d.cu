// filter3d.cu -- the 3D smoothing filter of every row from the training views (gsb200_filter3d_from_views; definition in
// include/gsb200.h).  One thread per row; the CTA stages the (view, object) entries -- the view's pose block for that object,
// K, W, H and f -- through shared memory in chunks of F3D_CHUNK, so any number of views and objects fits, and every thread
// tests its row against the staged entries of its own object.  The projection repeats the preprocess's float32 operations
// (this translation unit is compiled with -fmad=false like preprocess.cu), and the result is a min over views and a max over
// rows: bit-deterministic.  The largest seen d is an integer atomicMax on the bits of non-negative floats (they order as
// their bits), one per warp.
#include "common.cuh"

namespace gsb {

constexpr int F3D_THREADS = 256;
constexpr int F3D_CHUNK = 128;  // entries per round: 128 x 96 B = 12 KB of shared memory
constexpr int F3D_ENTRY = 24;   // floats per entry: T (12) | K00 K01 K02 K10 | K11 K12 W H | f object pad pad

struct Filter3dParams {
    long long N;
    const float *xyz;
    const signed char *invalid;
    const int *obj_id;
    int num_objects;
    long long num_entries;  // views x objects
    const PoseBlock *poses; // (V, objects): entry e = v * objects + o
    const float *K;         // (V, 3, 3)
    const int *size;        // (V, 2) {W, H}
    float near_plane;
    float sqrt_variance;
    float *filter3d;        // (N,) out: sqrt(variance) d, 0 for invalid rows, -1 for valid rows no view sees
    int *max_d_bits;        // the largest d of the seen rows, as int bits (0 = none seen)
};

__global__ void __launch_bounds__(F3D_THREADS) filter3d_views_kernel(const Filter3dParams p) {
    __shared__ __align__(16) float s_entry[F3D_CHUNK * F3D_ENTRY];
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool valid = i < p.N && p.invalid[i] == 0;
    float x = 0.0f, y = 0.0f, z = 0.0f;
    int ob = -1;
    if (valid) {
        x = p.xyz[3 * i];
        y = p.xyz[3 * i + 1];
        z = p.xyz[3 * i + 2];
        ob = p.obj_id[i];
    }
    float d_min = INFINITY;
    bool seen = false;
    for (long long e0 = 0; e0 < p.num_entries; e0 += F3D_CHUNK) {
        const int n = p.num_entries - e0 < F3D_CHUNK ? (int)(p.num_entries - e0) : F3D_CHUNK;
        __syncthreads();  // every thread is done with the previous chunk
        for (int k = threadIdx.x; k < n * F3D_ENTRY; k += blockDim.x) {
            const int e = k / F3D_ENTRY, w = k - e * F3D_ENTRY;
            const long long ge = e0 + e;
            const long long v = ge / p.num_objects;
            float val = 0.0f;
            if (w < 12) val = p.poses[ge].T[w];
            else if (w < 18) val = p.K[9 * v + (w - 12)];  // K00 K01 K02 K10 K11 K12
            else if (w < 20) val = (float)p.size[2 * v + (w - 18)];
            else if (w == 20) val = fmaxf(p.K[9 * v], p.K[9 * v + 4]);
            else if (w == 21) val = __int_as_float((int)(ge - v * p.num_objects));
            s_entry[k] = val;
        }
        __syncthreads();
        if (!valid) continue;
        for (int e = 0; e < n; ++e) {
            const float4 *E = reinterpret_cast<const float4 *>(s_entry + e * F3D_ENTRY);
            const float4 e5 = E[5];
            if (__float_as_int(e5.y) != ob) continue;
            const float4 t0 = E[0], t1 = E[1], t2 = E[2], k0 = E[3], k1 = E[4];
            // preprocess_body: pc = T (x, y, z, 1), uv = (K pc)[:2] / z
            const float pc0 = ((t0.x * x + t0.y * y) + t0.z * z) + t0.w * 1.0f;
            const float pc1 = ((t1.x * x + t1.y * y) + t1.z * z) + t1.w * 1.0f;
            const float pc2 = ((t2.x * x + t2.y * y) + t2.z * z) + t2.w * 1.0f;
            if (!(pc2 > p.near_plane && e5.x > 0.0f)) continue;
            const float u = ((k0.x * pc0 + k0.y * pc1) + k0.z * pc2) / pc2;
            const float v = ((k0.w * pc0 + k1.x * pc1) + k1.y * pc2) / pc2;
            const float Wf = k1.z, Hf = k1.w;
            if (u >= -0.15f * Wf && u <= 1.15f * Wf && v >= -0.15f * Hf && v <= 1.15f * Hf) {
                d_min = fminf(d_min, pc2 / e5.x);
                seen = true;
            }
        }
    }
    int bits = seen ? __float_as_int(d_min) : 0;
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) bits = max(bits, __shfl_xor_sync(0xffffffffu, bits, s));
    if ((threadIdx.x & 31) == 0 && bits > 0) atomicMax(p.max_d_bits, bits);
    if (i < p.N) p.filter3d[i] = !valid ? 0.0f : seen ? p.sqrt_variance * d_min : -1.0f;
}

// The valid rows no view sees get sqrt(variance) times the largest seen d (0 when no row is seen).
__global__ void __launch_bounds__(F3D_THREADS) filter3d_unseen_kernel(const Filter3dParams p) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.N) return;
    if (p.filter3d[i] < 0.0f) p.filter3d[i] = p.sqrt_variance * __int_as_float(*p.max_d_bits);
}

constexpr long long F3D_TEMP_HEAD = 256;  // the max word, then the pose blocks

static inline long long filter3d_temp_bytes(long long views, long long objects) {
    return F3D_TEMP_HEAD + views * objects * (long long)sizeof(PoseBlock);
}

static inline Filter3dParams filter3d_params(const GsbFilter3dViewsArgs &a) {
    Filter3dParams p;
    char *t = static_cast<char *>(a.temp);
    p.N = a.num_points;
    p.xyz = a.pointcloud;
    p.invalid = reinterpret_cast<const signed char *>(a.point_invalid_mask);
    p.obj_id = a.point_object_id;
    p.num_objects = a.num_objects;
    p.num_entries = (long long)a.num_views * a.num_objects;
    p.poses = reinterpret_cast<const PoseBlock *>(t + F3D_TEMP_HEAD);
    p.K = a.camera_intrinsics;
    p.size = a.camera_size;
    p.near_plane = a.near_plane;
    p.sqrt_variance = sqrtf(a.variance);
    p.filter3d = a.filter3d;
    p.max_d_bits = reinterpret_cast<int *>(t);
    return p;
}

#ifndef GSB_HOST_EMU  // tests/simt compiles the kernels above as host C++ under the SIMT emulator
int launch_filter3d_from_views(const GsbFilter3dViewsArgs &a, cudaStream_t stream) {
    const Filter3dParams p = filter3d_params(a);
    GSB_CUDA_CHECK(cudaMemsetAsync(p.max_d_bits, 0, sizeof(int), stream));
    int rc = launch_pose_blocks(a.q_pointcloud_camera, a.t_pointcloud_camera, (int)p.num_entries,
                                const_cast<PoseBlock *>(p.poses), stream);
    if (rc != GSB_OK || a.num_points <= 0) return rc;
    const long long blocks = (a.num_points + F3D_THREADS - 1) / F3D_THREADS;
    filter3d_views_kernel<<<(unsigned)blocks, F3D_THREADS, 0, stream>>>(p);
    GSB_CUDA_CHECK(cudaGetLastError());
    filter3d_unseen_kernel<<<(unsigned)blocks, F3D_THREADS, 0, stream>>>(p);
    GSB_CUDA_CHECK(cudaGetLastError());
    return GSB_OK;
}
#endif  // GSB_HOST_EMU

}  // namespace gsb

#ifndef GSB_HOST_EMU
extern "C" {

int64_t gsb200_filter3d_temp_bytes(int32_t num_views, int32_t num_objects) {
    return num_views < 1 || num_objects < 1 ? 0 : gsb::filter3d_temp_bytes(num_views, num_objects);
}

int gsb200_filter3d_from_views(const GsbFilter3dViewsArgs *a) {
    using gsb::set_error;
    if (!a) {
        set_error("filter3d_from_views: args is null");
        return GSB_EINVAL;
    }
    if (a->num_points < 0 || a->num_views < 1 || a->num_objects < 1) {
        set_error("filter3d_from_views: need num_points >= 0, num_views >= 1 and num_objects >= 1 (got %lld, %d, %d)",
                  (long long)a->num_points, a->num_views, a->num_objects);
        return GSB_EINVAL;
    }
    if ((long long)a->num_views * a->num_objects > (1LL << 30)) {
        set_error("filter3d_from_views: num_views x num_objects must be <= 2^30 (got %d x %d)", a->num_views, a->num_objects);
        return GSB_EUNSUPPORTED;
    }
    if (!(a->near_plane >= 0.0f && a->near_plane <= 3.402823466e38f) || !(a->variance >= 0.0f && a->variance <= 3.402823466e38f)) {
        set_error("filter3d_from_views: the near plane and the variance must be finite and >= 0 (got %g, %g)",
                  (double)a->near_plane, (double)a->variance);
        return GSB_EINVAL;
    }
    const void *ptrs[] = {a->pointcloud, a->point_invalid_mask, a->point_object_id, a->filter3d};
    bool bad = false;
    if (a->num_points > 0)
        for (const void *q : ptrs) bad = bad || q == nullptr;
    const void *views[] = {a->q_pointcloud_camera, a->t_pointcloud_camera, a->camera_intrinsics, a->camera_size};
    for (const void *q : views) bad = bad || q == nullptr || reinterpret_cast<uintptr_t>(q) % 4 != 0;
    const void *aligned4[] = {a->pointcloud, a->point_object_id, a->filter3d};
    for (const void *q : aligned4) bad = bad || reinterpret_cast<uintptr_t>(q) % 4 != 0;
    if (bad) {
        set_error("filter3d_from_views: null or not 4-byte aligned pointer");
        return GSB_EINVAL;
    }
    if (!a->temp || reinterpret_cast<uintptr_t>(a->temp) % 16 != 0 ||
        a->temp_bytes < gsb200_filter3d_temp_bytes(a->num_views, a->num_objects)) {
        set_error("filter3d_from_views: temp null, not 16-byte aligned or smaller than gsb200_filter3d_temp_bytes "
                  "(temp_bytes=%lld)", (long long)a->temp_bytes);
        return GSB_EINVAL;
    }
    return gsb::launch_filter3d_from_views(*a, static_cast<cudaStream_t>(a->stream));
}

}  // extern "C"
#endif  // GSB_HOST_EMU
