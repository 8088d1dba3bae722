// blend_bwd.cu -- backward of the blend (replaces gaussian_point_rasterisation_backward, GPCR:488-772).
//
// Kernel A (loop A, GPCR:531-705): one CTA per tile replays its splat list back-to-front.  The
// reference issues 11 global atomics per contributing (pixel, splat); here the 11 per-splat partials
// (d/duv x2, d/dcov x3, d/dcolour x3, d/dlogit, |d/duv|, pixel count) are reduced across the warp
// with a transposing butterfly (13 shuffles for all of them) and flushed with ONE 11-lane RED.ADD.F32
// per (warp patch, splat) -- per-warp culling (common.cuh) leaves ~2 of the 8 patches per (tile, splat).
// Kernel B (loop B, GPCR:708-772 + GPCR:1102-1125, 1167-1182): per in-frustum point chain rule to
// xyz / q / s / SH with the SH-band masking and the constant gradient factors fused in.
#include "blend_bwd.cuh"

namespace gsb {

// Reduce 11 per-lane values across the warp with 13 shuffles (transposing butterfly: at every stage a lane hands
// one half of its live values to its partner and keeps the other half, 11 -> 6 -> 3 -> 2 -> 1; the odd value of a
// stage is summed on both sides).  On return v[0] of lane l holds the warp total of value index
// reduce11_slot(l); the lanes for which reduce11_writer(l) is true cover 0..10 exactly once.
__device__ __forceinline__ void warp_transpose_reduce11(float (&v)[11], int lane) {
    {
        const bool hi = lane & 16;  // keeps values 6..10 (and a duplicate of 5), partner keeps 0..5
#pragma unroll
        for (int i = 0; i < 5; ++i) {
            const float send = hi ? v[i] : v[i + 6];
            const float keep = hi ? v[i + 6] : v[i];
            v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
        }
        v[5] += __shfl_xor_sync(0xffffffffu, v[5], 16);
    }
    {
        const bool hi = lane & 8;  // slots 3..5 vs 0..2
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const float send = hi ? v[i] : v[i + 3];
            const float keep = hi ? v[i + 3] : v[i];
            v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
        }
    }
    {
        const bool hi = lane & 4;  // slot 2 vs slot 0; slot 1 on both sides
        const float send = hi ? v[0] : v[2];
        const float keep = hi ? v[2] : v[0];
        v[0] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
        v[1] += __shfl_xor_sync(0xffffffffu, v[1], 4);
    }
    {
        const bool hi = lane & 2;  // slot 1 vs slot 0
        const float send = hi ? v[0] : v[1];
        const float keep = hi ? v[1] : v[0];
        v[0] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
    }
    v[0] += __shfl_xor_sync(0xffffffffu, v[0], 1);
}
__device__ __forceinline__ int reduce11_slot(int lane) {
    const int s2 = (lane & 2) ? 1 : ((lane & 4) ? 2 : 0);
    const int s1 = s2 + ((lane & 8) ? 3 : 0);
    return (lane & 16) ? (s1 == 5 ? 5 : s1 + 6) : s1;
}
__device__ __forceinline__ bool reduce11_writer(int lane) {
    if (lane & 1) return false;
    if ((lane & 2) && (lane & 4)) return false;         // slot 1 is duplicated over bit 2
    if ((lane & 16) && (lane & 8) && !(lane & 2) && (lane & 4)) return false;  // duplicate of value 5 in the upper half
    return true;
}


#ifndef GSB_BWD_MIN_BLOCKS
#define GSB_BWD_MIN_BLOCKS 4
#endif
// STATS = false (GSB_FLAG_NO_HOOK_STATS, opt-in): the |d/duv| magnitude, the affected-pixel count and the per-pixel magnitude
// image -- read only by a backward hook, the reference's need_extra_info (GPCR:521, 690-704) -- are not computed; slots 9 and
// 10 of the butterfly then carry zeros.
template <bool EXACT_EXP, bool STATS = true>
__global__ void __launch_bounds__(GSB_TILE_PIXELS, GSB_BWD_MIN_BLOCKS)
blend_backward_kernel(const BlendBwdParams p) {
    // double-buffered staging area: [buf][plane][splat]; planes: u v a b | c rescale opacity depth | r g b radius
    __shared__ float4 s_rec[2 * 3 * GSB_TILE_PIXELS];
    __shared__ int s_off[2][GSB_TILE_PIXELS];
    constexpr int PLANE = GSB_TILE_PIXELS * 16;
    __shared__ unsigned int s_bits[2][8][8];  // [buf][consumer warp patch][loader warp]
    __shared__ int s_max_last;

    const int tile = blockIdx.x;
    const int tu = tile % p.tiles_x, tv = tile / p.tiles_x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int pu = tu * GSB_TILE_WIDTH + (warp & 1) * 8 + (lane & 7);
    const int pv = tv * GSB_TILE_HEIGHT + (warp >> 1) * 4 + (lane >> 3);
    const float px = (float)pu + 0.5f, py = (float)pv + 0.5f;
    const float tile_x0 = (float)(tu * GSB_TILE_WIDTH), tile_y0 = (float)(tv * GSB_TILE_HEIGHT);
    const size_t pix = (size_t)pv * p.W + pu;
    const int start = p.tile_start[tile];

    const int last = p.last_effective[pix];
    float T = 1.0f - p.acc_alpha[pix];  // GPCR:559-560
    float w0 = 0.0f, w1 = 0.0f, w2 = 0.0f;
    const float g0 = p.grad_image[3 * pix], g1 = p.grad_image[3 * pix + 1], g2 = p.grad_image[3 * pix + 2];
    float mag0 = 0.0f, mag1 = 0.0f;
    const unsigned int sa = smem_u32(s_rec);
    const int red_slot = reduce11_slot(lane);
    const bool red_writer = reduce11_writer(lane);

    // deepest effective splat of this warp's patch and of the whole tile (GPCR:609-610: nothing at or
    // behind a pixel's last effective offset contributes to it)
    int warp_last = last;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) warp_last = max(warp_last, __shfl_xor_sync(0xffffffffu, warp_last, d));
    if (tid == 0) s_max_last = start;
    __syncthreads();
    if (lane == 0) atomicMax(&s_max_last, warp_last);
    __syncthreads();
    const int end = min(p.tile_end[tile], s_max_last);

    // One barrier per batch (double-buffered staging, see blend_fwd.cu).
    int buf = 0;
    for (int block_end = end; block_end > start; block_end -= GSB_TILE_PIXELS, buf ^= 1) {
        const int block_start = max(block_end - GSB_TILE_PIXELS, start);
        float4 *const s_r0 = s_rec + buf * 3 * GSB_TILE_PIXELS;
        float4 *const s_r1 = s_r0 + GSB_TILE_PIXELS, *const s_r2 = s_r0 + 2 * GSB_TILE_PIXELS;
        {
            const int idx = block_end - 1 - tid;  // element j <-> sorted index block_end-1-j
            unsigned int mask = 0;
            if (idx >= block_start) {
                const int o = __ldg(&p.sorted_vals[idx]);
                const float4 *rec = p.records + 3 * (size_t)o;
                const float4 r0 = __ldg(rec), r1 = __ldg(rec + 1);
                s_r0[tid] = r0;
                // fast path: the loop needs rescale*opacity and 1-opacity, not the two factors
                s_r1[tid] = EXACT_EXP ? r1 : make_float4(r1.x, r1.y * r1.z, 1.0f - r1.z, r1.w);
                s_r2[tid] = __ldg(rec + 2);
                s_off[buf][tid] = o;
                mask = splat_patch_mask(r0.x, r0.y, r0.z, r0.w, r1.x, r1.y * r1.z, tile_x0, tile_y0);
            }
#pragma unroll
            for (int w = 0; w < 8; ++w) {
                const unsigned int bits = __ballot_sync(0xffffffffu, (mask >> w) & 1u);
                if (lane == 0) s_bits[buf][w][warp] = bits;
            }
        }
        __syncthreads();
        const unsigned int sb = sa + buf * (3 * PLANE);
        if (block_start < warp_last) {  // otherwise every splat of this batch is behind the whole patch
            // element j <-> sorted index block_end-1-j: the first `skip` elements of the batch lie at or behind the
            // patch's deepest effective splat and are dropped from the bit lists wholesale (warp-uniform)
            const int skip = block_end - warp_last;
#pragma unroll 1
            for (int lw = skip > 0 ? (skip >> 5) : 0; lw < 8; ++lw) {
                unsigned int bits = s_bits[buf][warp][lw];
                if (skip > lw * 32) bits &= ~((1u << (skip - lw * 32)) - 1u);  // 0 < skip - 32 lw < 32 here
                while (bits) {
                    const int j = lw * 32 + __ffs(bits) - 1;
                    bits &= bits - 1;
                    const int idx = block_end - 1 - j;
                    float v[11];
                    bool contributes;
                    // Branch-free: every lane evaluates the splat; lanes that do not contribute (behind their
                    // last effective splat, or alpha < 1/255) get zero weights, so all partials vanish and the
                    // pixel state is left untouched by predicated selects.
                    {
                        const unsigned int ja = sb + j * 16;
                        const float4 r0 = lds128<0>(ja);          // u v a b
                        const float4 r1 = lds128<PLANE>(ja);      // c rescale opacity depth
                        const float4 r2 = lds128<2 * PLANE>(ja);  // r g b radius
                        const float d0 = px - r0.x, d1 = py - r0.y;
                        const float q0 = r0.z * d0 + r0.w * d1;
                        const float q1 = r0.w * d0 + r1.x * d1;
                        if (EXACT_EXP) {
                            const float gp = expf(-0.5f * (d0 * q0 + d1 * q1)) * r1.y;
                            const float opa = r1.z;
                            const float prod_alpha = gp * opa;
                            contributes = (idx < last) && (prod_alpha >= 1.0f / 255.0f);
                            const float alpha = fminf(prod_alpha, 0.99f);
                            const float inv = 1.0f / (1.0f - alpha);
                            const float Tn = T * inv;
                            const float aT = contributes ? alpha * Tn : 0.0f;
                            const float a_grad = contributes ? (r2.x * Tn - w0 * inv) * g0 + (r2.y * Tn - w1 * inv) * g1 +
                                                                   (r2.z * Tn - w2 * inv) * g2
                                                             : 0.0f;
                            T = contributes ? Tn : T;
                            w0 = fmaf(r2.x, aT, w0);
                            w1 = fmaf(r2.y, aT, w1);
                            w2 = fmaf(r2.z, aT, w2);
                            const float G = a_grad * opa * gp;
                            const float vs0 = G * q0, vs1 = G * q1;
                            if (STATS) {
                                mag0 += fabsf(vs0);
                                mag1 += fabsf(vs1);
                            }
                            v[0] = vs0;
                            v[1] = vs1;
                            v[2] = vs0 * q0;  // the 1/2 of UT:345 is applied once per point in the epilogue
                            v[3] = vs0 * q1;
                            v[4] = vs1 * q1;
                            v[5] = aT * g0;
                            v[6] = aT * g1;
                            v[7] = aT * g2;
                            v[8] = a_grad * gp * (1.0f - opa) * opa;
                            v[9] = STATS ? sqrtf(vs0 * vs0 + vs1 * vs1) : 0.0f;
                        } else {
                            // r1 = c | rescale*opacity | 1-opacity | depth.  The colour recursion of GPCR:653-657,
                            // sum_c (col_c T - w_c/(1-a)) g_c, is carried as ONE scalar: with cg = sum_c col_c g_c and
                            // w0 = sum_c w_c g_c it is  cg T - w0/(1-a),  and w0 += cg a T.
                            // alpha exactly as the forward computes it (fast_alpha on the forward's pre-scaled conic, common.cuh): both
                            // passes take the alpha >= 1/255 decision on identical bits
                            const float P = fast_alpha(d0, d1, (-0.5f * GSB_L2E) * r0.z, -GSB_L2E * r0.w,
                                                       (-0.5f * GSB_L2E) * r1.x, r1.y);
                            contributes = (idx < last) && (P >= 1.0f / 255.0f);
                            const float alpha = fminf(P, 0.99f);
                            const float inv = rcp_approx(1.0f - alpha);
                            const float Tn = T * inv;
                            const float aT = contributes ? alpha * Tn : 0.0f;
                            const float cg = fmaf(r2.z, g2, fmaf(r2.y, g1, r2.x * g0));
                            const float a_grad = contributes ? fmaf(cg, Tn, -(w0 * inv)) : 0.0f;
                            T = contributes ? Tn : T;
                            w0 = fmaf(cg, aT, w0);
                            const float G = a_grad * P;  // d L / d gaussian exponent weight: a_grad * opacity * p
                            const float vs0 = G * q0, vs1 = G * q1;
                            if (STATS) {
                                mag0 += fabsf(vs0);
                                mag1 += fabsf(vs1);
                            }
                            v[0] = vs0;
                            v[1] = vs1;
                            v[2] = vs0 * q0;
                            v[3] = vs0 * q1;
                            v[4] = vs1 * q1;
                            v[5] = aT * g0;
                            v[6] = aT * g1;
                            v[7] = aT * g2;
                            v[8] = G * r1.z;  // a_grad * p * opacity * (1 - opacity)
                            v[9] = STATS ? sqrt_approx(vs0 * vs0 + vs1 * vs1) : 0.0f;
                        }
                        v[10] = (STATS && contributes) ? 1.0f : 0.0f;
                    }
                    if (lane == 0) GSB_EMU_COUNT(EC_BF_VISITS, 1);
                    GSB_EMU_COUNT(EC_BF_PAIRS, contributes ? 1 : 0);
                    if (__any_sync(0xffffffffu, contributes)) {
                        if (lane == 0) GSB_EMU_COUNT(EC_BF_VISITS_ANY, 1);
                        // 11 partials of this (warp, splat) -> 11 lanes -> one RED.ADD.F32 row update
                        warp_transpose_reduce11(v, lane);
                        if (red_writer && (STATS || red_slot < 9))
                            atomicAdd(p.accum + (size_t)s_off[buf][j] * GSB_ACCUM_FLOATS + red_slot, v[0]);
                    }
                }
            }
        }
    }
    if (STATS) {
        p.mag_image[2 * pix] = mag0;  // GPCR:700-704
        p.mag_image[2 * pix + 1] = mag1;
    }
}

#ifndef GSB_HOST_EMU
static BlendBwdParams make_blend_bwd_params(const GsbBackwardArgs &a, const Workspace &ws);

int launch_blend_backward_work(const GsbBackwardArgs &a, const Workspace &ws, unsigned long long *counters_dev,
                               cudaStream_t stream) {
    BlendBwdParams p = make_blend_bwd_params(a, ws);
    p.work_counters = counters_dev;
    const int tiles = p.tiles_x * (a.camera_height / GSB_TILE_HEIGHT);
    if (tiles <= 0) return GSB_OK;
    return launch_blend_backward_count(p, tiles, stream);
}

static BlendBwdParams make_blend_bwd_params(const GsbBackwardArgs &a, const Workspace &ws) {
    BlendBwdParams p;
    p.H = a.camera_height;
    p.W = a.camera_width;
    p.tiles_x = a.camera_width / GSB_TILE_WIDTH;
    p.tile_start = ws.tile_start;
    p.tile_end = ws.tile_end;
    p.sorted_vals = ws.vals_b;  // the sort always ends in b
    p.records = ws.records;
    p.grad_image = a.grad_rasterized_image;
    p.acc_alpha = a.pixel_accumulated_alpha;
    p.last_effective = a.pixel_offset_of_last_effective_point;
    p.accum = a.accum;
    p.mag_image = a.magnitude_grad_viewspace_on_image;
    p.work_counters = nullptr;
    p.grad_depth = nullptr;
    p.depth = nullptr;
    p.grad_alpha = nullptr;
    return p;
}

int launch_blend_backward(const GsbBackwardArgs &a, const Workspace &ws, cudaStream_t stream, const float *grad_depth,
                          const float *depth, const float *grad_alpha, const GsbExtraFeatureArgs *ext, bool wrap) {
    BlendBwdParams p;
    p.H = a.camera_height;
    p.W = a.camera_width;
    p.tiles_x = a.camera_width / GSB_TILE_WIDTH;
    p.tile_start = ws.tile_start;
    p.tile_end = ws.tile_end;
    p.sorted_vals = ws.vals_b;  // the sort always ends in b
    p.records = ws.records;
    p.grad_image = a.grad_rasterized_image;
    p.acc_alpha = a.pixel_accumulated_alpha;
    p.last_effective = a.pixel_offset_of_last_effective_point;
    p.accum = a.accum;
    p.mag_image = a.magnitude_grad_viewspace_on_image;
    p.work_counters = nullptr;
    p.grad_depth = grad_depth;
    p.depth = depth;
    p.grad_alpha = grad_alpha;
    const BlendFeatureParams feat{ext ? ext->channels : 0, ws.point_id, ext ? ext->features : nullptr,
                                  ext ? ext->grad_rasterized : nullptr, ext ? ext->grad_features : nullptr};
    const int tiles = p.tiles_x * (a.camera_height / GSB_TILE_HEIGHT);
    if (tiles <= 0) return GSB_OK;
    if (a.flags & GSB_FLAG_BACKWARD_TRANSPOSED)  // experimental, see blend_bwd_transposed.cu
        return launch_blend_backward_transposed(p, tiles, (a.flags & GSB_FLAG_EXACT_EXP) != 0,
                                                (a.flags & GSB_FLAG_NO_HOOK_STATS) == 0, stream, grad_depth != nullptr,
                                                grad_alpha != nullptr, ext ? &feat : nullptr, wrap);
    const bool exact = (a.flags & GSB_FLAG_EXACT_EXP) != 0;
    if (a.flags & GSB_FLAG_NO_HOOK_STATS) {  // opt-in
        if (exact) blend_backward_kernel<true, false><<<tiles, GSB_TILE_PIXELS, 0, stream>>>(p);
        else blend_backward_kernel<false, false><<<tiles, GSB_TILE_PIXELS, 0, stream>>>(p);
    } else if (exact) {
        blend_backward_kernel<true><<<tiles, GSB_TILE_PIXELS, 0, stream>>>(p);
    } else {
        blend_backward_kernel<false><<<tiles, GSB_TILE_PIXELS, 0, stream>>>(p);
    }
    GSB_CUDA_CHECK(cudaGetLastError());
    return GSB_OK;
}
#endif  // GSB_HOST_EMU

// ------------------------------------------------------------------ loop B + P4
// Real SH basis up to band 3 along the (un-normalised) direction (dx, dy, dz)  (SH:10-32; GPCR:731-732, 749)
__device__ __forceinline__ void sh_basis(float dx, float dy, float dz, float (&sh)[16]) {
    const float dinv = 1.0f / sqrtf(dx * dx + dy * dy + dz * dz);
    dx *= dinv; dy *= dinv; dz *= dinv;
    sh[0] = 0.28209479177387814f;
    sh[1] = -0.48860251190291987f * dy;
    sh[2] = 0.48860251190291987f * dz;
    sh[3] = -0.48860251190291987f * dx;
    sh[4] = 1.0925484305920792f * dx * dy;
    sh[5] = -1.0925484305920792f * dy * dz;
    sh[6] = 0.94617469575755997f * dz * dz - 0.31539156525251999f;
    sh[7] = -1.0925484305920792f * dx * dz;
    sh[8] = 0.54627421529603959f * dx * dx - 0.54627421529603959f * dy * dy;
    sh[9] = 0.59004358992664352f * dy * (-3.0f * dx * dx + dy * dy);
    sh[10] = 2.8906114426405538f * dx * dy * dz;
    sh[11] = 0.45704579946446572f * dy * (1.0f - 5.0f * dz * dz);
    sh[12] = 0.3731763325901154f * dz * (5.0f * dz * dz - 3.0f);
    sh[13] = 0.45704579946446572f * dx * (1.0f - 5.0f * dz * dz);
    sh[14] = 1.4453057213202769f * dz * (dx * dx - dy * dy);
    sh[15] = 0.59004358992664352f * dx * (-dx * dx + 3.0f * dy * dy);
}

struct PointsBwdParams {
    long long N;
    const int *point_offset;
    const float4 *records;
    const float *point_in_camera;
    const float *accum;
    const PoseBlock *poses;
    const float *xyz;
    const float *features;
    const int *obj_id;
    const float *t_pc_cam;
    const float *K;
    int first_cleared;  // first SH coefficient index whose gradient is zeroed (GPCR:1167-1182)
    float q_f, s_f, a_f, c_f, h_f;
    float *grad_xyz;
    float *grad_feat;
    // optional: the densification controller's accumulators, updated in this epilogue (GaussianPointAdaptiveController.py:130-143)
    int *ctl_num_in_camera;     // (N) or nullptr = not fused
    int *ctl_num_pixels;        // (N)
    float *ctl_vs_grad;         // (N)   accumulated_view_space_position_gradients
    float *ctl_vs_grad_avg;     // (N)   accumulated_view_space_position_gradients_avg
    float *ctl_pos_grad;        // (N,3) accumulated_position_gradients
    float *ctl_pos_grad_norm;   // (N)   accumulated_position_gradients_norm
    const long long *skip_flag; // optional device flag (the frame's key-capacity overflow counter): non-zero = leave the
                                //   controller accumulators alone (fused train step: the whole step becomes a no-op)
    float *grad_sum_compact;    // COMPACT: (N,12) xyz(3) q(4) s(3) logit(1) pad -- the columns that simply add up over views
    float *grad_color_compact;  // COMPACT: (N,3) d L / d (SH colour argument), per VIEW (its SH basis depends on the camera centre)
};

#ifndef GSB_POINTS_THREADS
#define GSB_POINTS_THREADS 128
#endif
constexpr int PT_ROW = 60;  // staged feature row stride in floats: 16-B aligned, float4 stores of 8 lanes hit 32 banks
constexpr int PT_ROW_COMPACT = 20;  // COMPACT: 16 staged floats per row, same bank property
// COMPACT = true (GSB_FLAG_COMPACT_GRADS, the view-parallel exchange of parallel.py): instead of the dense (N,3) / (N,56)
// gradients the kernel writes, per scene row, the 11 values that add up over views -- xyz(3) q(4) s(3) logit(1), factors
// applied -- and the 3 colour-argument gradients that must stay per view: the 48 SH gradients of a view are their outer product
// with the view's SH basis, which gsb200_expand_view_gradients rebuilds AFTER the exchange (14 instead of 59 floats per row
// cross NVLink, and this kernel writes 60 instead of 236 bytes per row).
// DEPTH = true (gsb200_backward_with_depth): word 11 of the accumulator row is dL/dz of the point's camera-space depth
// (blend_bwd_transposed.cu), and z = W[2,:] xyz + t adds it to dL/dxyz along the third row of W -- before gx feeds the
// dense gradient, the controller epilogue or the compact row.
// POSE = true (gsb200_backward_pose): each in-camera point also forms its 12 pose values -- dL/dW (9, row-major) and
// dL/dtw (3) of its object's T = [W | tw] -- which the warp sums per object (fixed butterfly order) into the per-warp rows
// s_pose[warp][object][12]; after the loop the CTA adds its warps' rows in warp order into its partial row block
// pose_partials[blockIdx.x][object][12].  pose_finish_kernel adds the blocks in block order: no float atomics anywhere.
// INTR = true (gsb200_backward_calib): each in-camera point also forms its 6 intrinsics values -- dL/dK of rows 0 and 1,
// row-major -- which the warp sums (fixed butterfly order, all objects together: a frame has one K) into the per-warp row
// s_intr[warp][6]; after the loop the CTA adds its warps' rows in warp order into intr_partials[blockIdx.x][6], and
// intrinsics_finish_kernel adds the blocks in block order.
constexpr int POSE_VALUES = 12;
constexpr int INTR_VALUES = 6;
// B0, B1: the rows of G U Sigma (Sigma = M M^T, M = R diag(es)), so that dL/dU = 2 [B0; B1] for U = J W
__device__ __forceinline__ void weighted_u_sigma(const float *U, const float *R, const float *es, float g00, float g01,
                                                 float g11, float *B0, float *B1) {
    float UM[6];  // U M, M = R diag(es)
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            UM[a * 3 + j] = (U[a * 3] * R[j] + U[a * 3 + 1] * R[3 + j] + U[a * 3 + 2] * R[6 + j]) * es[j];
#pragma unroll
    for (int c = 0; c < 3; ++c) {  // G U Sigma = G (U M) M^T
        const float A0 = UM[0] * (R[c * 3] * es[0]) + UM[1] * (R[c * 3 + 1] * es[1]) + UM[2] * (R[c * 3 + 2] * es[2]);
        const float A1 = UM[3] * (R[c * 3] * es[0]) + UM[4] * (R[c * 3 + 1] * es[1]) + UM[5] * (R[c * 3 + 2] * es[2]);
        B0[c] = g00 * A0 + g01 * A1;
        B1[c] = g01 * A0 + g11 * A1;
    }
}
// LENS = true (gsb200_backward_lens): the frame was projected through lens_distort (common.cuh), so d uv / d pc = K[:2,:2] D P
// replaces the pinhole projection Jacobian and J = diag(fx, fy) D P replaces the pinhole J inside Sigma' (D at the point's
// (xn, yn), detached like J).  Non-compact.  With POSE (gsb200_backward_lens_calib), J is a full 2x3 matrix:
// dL/dW[r] = gp_r xyz + 2 sum_a J[a][r] B_a.  With INTR: dL/dK[r][c] = guv_r (xd, yd, 1)_c, and fx, fy enter J through
// diag(fx, fy): dL/dK[0][0] += 2 B0 . (D P W)[0], dL/dK[1][1] += 2 B1 . (D P W)[1].
// LGRAD = true (gsb200_backward_lens_grad, with LENS): each in-camera point also forms its 5 coefficient values
// (lens_coefficient_grad, common.cuh), which the warp sums (fixed butterfly order, all objects together: a frame has one lens)
// into the per-warp row s_lgrad[warp][5]; after the loop the CTA adds its warps' rows in warp order into
// lgrad_partials[blockIdx.x][5], and lens_grad_finish_kernel adds the blocks in block order.
// RS = true (gsb200_backward_rolling_shutter): the frame was rendered through a rolling shutter (include/gsb200.h), so the
// point's row time tau = rs.row_time[id] (written by the forward; detached) gives W_eff = Rd(tau) W, which replaces W in
// d uv / d xyz, the depth term and U = J W_eff; point_in_camera already holds pc(tau).  Non-compact, without POSE / INTR /
// LGRAD; with or without LENS.
// MGRAD = true (with RS and rs_grad): each in-camera point also forms its 6 motion values (rolling_shutter_grad, common.cuh),
// which the warp sums (fixed butterfly order, all objects together: a frame has one motion) into the per-warp row
// s_mgrad[warp][6]; after the loop the CTA adds its warps' rows in warp order into mgrad_partials[blockIdx.x][6], and
// rolling_shutter_grad_finish_kernel adds the blocks in block order.
// FILTER = true (gsb200_backward_filter3d): the frame was rendered with the 3D smoothing filter sigma = fmaxf(filter3d[id], 0)
// (include/gsb200.h): s^_j = sqrt(e_j + sigma^2), e_j = exp(s_j)^2, replaces exp(s_j) in M = R diag(s^), and
//   dL/ds_j = (sum_l dM_lj R_lj) s^_j (e_j / e^_j) + G_a sigma^2 / e^_j,   G_a = glogit / fl(1 - o)
// where o is the record's raw opacity r1.z (the float the blend multiplied by); the compensation term is dropped where
// fl(1 - o) = 0.  dL/dlogit is unchanged: the compensation c does not depend on the logit.  Non-compact, without POSE / INTR /
// LGRAD / MGRAD.
// BLUR = true (gsb200_backward_motion_blur): the frame was rendered with the exposure motion m_b = blur.motion
// (include/gsb200.h): the conic was (Sigma_d + B)^-1 with B = d d^T / 12, d = Jp (v + w x pc) (detached, from dj and
// point_in_camera), and the rescale slot carried c_b.  G reaches Sigma' unchanged (B is additive), plus the compensation's
// G_a/2 (Sigma_d^-1 - (Sigma_d + B)^-1) with G_a = glogit / fl(1 - o) (dropped where fl(1 - o) = 0), before V = U^T G U
// (motion_blur_grad, common.cuh).  A view with m_b = 0 takes the un-blurred arithmetic.  Non-compact, without POSE / INTR /
// LGRAD / MGRAD / FILTER; with or without LENS and RS.
// BGRAD = true (with BLUR and blur_grad): each in-camera point also forms dL/dv = g and dL/dw = pc x g with g = Jp^T dL/dd,
// which go through the rows of MGRAD: s_mgrad, mgrad_partials and rolling_shutter_grad_finish_kernel.
// DEFOCUS = true (with BLUR; gsb200_backward_defocus): B also carries the thin lens' B_d = beta M M^T (include/gsb200.h; beta
// detached, at pcz).  With G_B = G - G_a/2 (Sigma_d + B)^-1 (blur_cov_grad, common.cuh), dL/dSigma' is that of BLUR with this
// B.  A view with a = 0 takes the arithmetic without defocus.  Not with BGRAD.
// DGRAD = true (with DEFOCUS and defocus_grad): each in-camera point also forms dL/da = dL/dbeta a (rho - 1/z)^2 / 8 and
// dL/drho = dL/dbeta a^2 (rho - 1/z) / 8 with dL/dbeta = <G_B, M M^T>, in the first two values of the rows of MGRAD.
constexpr int LENS_GRAD_VALUES = 5;
constexpr int RS_GRAD_VALUES = 6;
// EQUI = true (gsb200_backward_equirect): the frame is an equirectangular panorama (include/gsb200.h): d uv / d pc and the J
// of Sigma' are both equirect_jacobian at point_in_camera (J detached, as for every model), and with DEPTH word 11 is dL/dr
// of the ray distance, which enters pc along pc / r.  Non-compact, without any other camera path or gradient.
// ORTHO = true (gsb200_backward_ortho): the frame is an orthographic view (include/gsb200.h): d uv / d pc and the J of Sigma'
// are both K[:2,:2] [I 0], exact (J does not depend on pc), the depth term is the pinhole's along z, and the SH basis is taken
// along row 2 of W.  With POSE, J enters dL/dW through all four of its entries: dL/dW[r] = gp_r xyz + 2 sum_a J[a][r] B_a.  With
// INTR: dL/dK[r][c] = guv_r (x, y, 1)_c + 2 sum_j B_r[j] W[c][j] for c in {0, 1}.  Non-compact; with or without DEPTH, FILTER,
// POSE and INTR (FILTER never with POSE or INTR); without the other camera paths.
template <bool COMPACT, bool DEPTH, bool POSE, bool INTR = false, bool LENS = false, bool LGRAD = false, bool RS = false,
          bool MGRAD = false, bool FILTER = false, bool BLUR = false, bool BGRAD = false, bool DEFOCUS = false,
          bool DGRAD = false, bool EQUI = false, bool ORTHO = false>
__device__ __forceinline__ void backward_points_body(const PointsBwdParams p, float *s_pose, float *pose_partials,
                                                     int num_objects, float *s_intr = nullptr,
                                                     float *intr_partials = nullptr, const LensParams lens = LensParams(),
                                                     float *s_lgrad = nullptr, float *lgrad_partials = nullptr,
                                                     const RsParams rs = RsParams(), float *s_mgrad = nullptr,
                                                     float *mgrad_partials = nullptr, const float *filter3d = nullptr,
                                                     const BlurParams blur = BlurParams(),
                                                     const DefocusParams defocus = DefocusParams()) {
    static_assert(!LENS || !COMPACT, "the lens gradient is implemented for the dense rows alone");
    static_assert(!LGRAD || LENS, "the coefficient gradient needs the lens path");
    static_assert(!RS || (!COMPACT && !POSE && !INTR && !LGRAD), "the rolling shutter is implemented for the dense rows alone");
    static_assert(!MGRAD || RS, "the motion gradient needs the rolling-shutter path");
    static_assert(!FILTER || (!COMPACT && !POSE && !INTR && !LGRAD && !MGRAD),
                  "the 3D filter is implemented for the dense rows without camera gradients");
    static_assert(!BLUR || (!COMPACT && !POSE && !INTR && !LGRAD && !MGRAD && !FILTER),
                  "the motion blur is implemented for the dense rows without other camera gradients or the 3D filter");
    static_assert(!BGRAD || BLUR, "the exposure-motion gradient needs the motion-blur path");
    static_assert(!DEFOCUS || (BLUR && !BGRAD), "the defocus runs on the motion-blur path, without the exposure-motion gradient");
    static_assert(!DGRAD || DEFOCUS, "the defocus gradient needs the defocus path");
    static_assert(!EQUI || (!COMPACT && !POSE && !INTR && !LENS && !RS && !FILTER && !BLUR),
                  "the panorama is implemented for the dense rows without the other camera paths");
    static_assert(!ORTHO || (!COMPACT && !LENS && !RS && !BLUR && !EQUI),
                  "the orthographic view is implemented for the dense rows without the other camera paths");
    constexpr bool CAM6 = MGRAD || BGRAD || DGRAD;  // the rows of a camera gradient (rolling shutter, exposure or defocus)
    // One thread per scene row: rows outside the frustum get their zeros here (no separate memset of the
    // dense (N,3)/(N,56) gradients), rows inside get the chain rule.  A warp owns 32 consecutive rows, i.e. one
    // contiguous 7 KB piece of the (N,56) gradient and 384 B of the (N,3) one: each lane stages its row in
    // shared memory and the warp then streams the piece out with full 512-B stores (a lane writing its own
    // 224-B row directly touches 32 different lines per store instruction and stalls on the LSU queue).
    constexpr int ROW = COMPACT ? PT_ROW_COMPACT : PT_ROW;
    __shared__ __align__(16) float s_feat[GSB_POINTS_THREADS / 32][32 * ROW];
    __shared__ float s_xyz[GSB_POINTS_THREADS / 32][96];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float *const my_feat = &s_feat[warp][lane * ROW];
    float *const my_xyz = &s_xyz[warp][lane * 3];
    float *const my_pose = POSE ? s_pose + warp * (num_objects * POSE_VALUES) : nullptr;
    if (POSE) {
        for (int k = lane; k < num_objects * POSE_VALUES; k += 32) my_pose[k] = 0.0f;
        __syncwarp();
    }
    float *const my_intr = INTR ? s_intr + warp * INTR_VALUES : nullptr;
    if (INTR) {
        if (lane < INTR_VALUES) my_intr[lane] = 0.0f;
        __syncwarp();
    }
    float *const my_lgrad = LGRAD ? s_lgrad + warp * LENS_GRAD_VALUES : nullptr;
    if (LGRAD) {
        if (lane < LENS_GRAD_VALUES) my_lgrad[lane] = 0.0f;
        __syncwarp();
    }
    float *const my_mgrad = CAM6 ? s_mgrad + warp * RS_GRAD_VALUES : nullptr;
    if (CAM6) {
        if (lane < RS_GRAD_VALUES) my_mgrad[lane] = 0.0f;
        __syncwarp();
    }
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long base = (long long)blockIdx.x * blockDim.x + warp * 32; base < p.N; base += stride) {
      const long long id = base + lane;
      const int o = id < p.N ? p.point_offset[id] : -1;
      float pv[POSE ? POSE_VALUES : 1];
      int pose_obj = -1;
      float iv[INTR ? INTR_VALUES : 1];  // zero for rows outside the frustum
      if (INTR) {
#pragma unroll
          for (int k = 0; k < INTR_VALUES; ++k) iv[k] = 0.0f;
      }
      float lv[LGRAD ? LENS_GRAD_VALUES : 1];  // zero for rows outside the frustum
      if (LGRAD) {
#pragma unroll
          for (int k = 0; k < LENS_GRAD_VALUES; ++k) lv[k] = 0.0f;
      }
      float mv[CAM6 ? RS_GRAD_VALUES : 1];  // zero for rows outside the frustum
      if (CAM6) {
#pragma unroll
          for (int k = 0; k < RS_GRAD_VALUES; ++k) mv[k] = 0.0f;
      }
      if (o < 0) {
          if (!COMPACT) { my_xyz[0] = 0.0f; my_xyz[1] = 0.0f; my_xyz[2] = 0.0f; }
#pragma unroll
          for (int k = 0; k < (COMPACT ? 4 : GSB_FEATURE_DIM / 4); ++k)
              reinterpret_cast<float4 *>(my_feat)[k] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
      } else {
        const float4 *accp = reinterpret_cast<const float4 *>(p.accum + (size_t)o * GSB_ACCUM_FLOATS);
        const float4 a0 = accp[0], a1 = accp[1], a2 = accp[2];
        // a0 = guv.x guv.y g00 g01 | a1 = g11 gr gg gb | a2 = glogit mag n pad
        const float4 r2 = __ldg(p.records + 3 * (size_t)o + 2);  // r g b radius
        const float pcx = p.point_in_camera[3 * o], pcy = p.point_in_camera[3 * o + 1],
                    pcz = p.point_in_camera[3 * o + 2];
        const int ob = p.obj_id[id];
        const PoseBlock *pb = p.poses + ob;
        float Wm[9] = {pb->T[0], pb->T[1], pb->T[2], pb->T[4], pb->T[5], pb->T[6], pb->T[8], pb->T[9], pb->T[10]};
        float Kc[9];
#pragma unroll
        for (int k = 0; k < 9; ++k) Kc[k] = __ldg(&p.K[k]);
        const float x = p.xyz[3 * (size_t)id], y = p.xyz[3 * (size_t)id + 1], z = p.xyz[3 * (size_t)id + 2];
        const float4 *frow = reinterpret_cast<const float4 *>(p.features + (size_t)GSB_FEATURE_DIM * id);
        const float4 qv = __ldg(frow);
        const float4 sv = __ldg(frow + 1);  // s0 s1 s2 logit
        float Wo[9], Rd[9], tau = 0.0f;  // RS: the object's W, Rd(tau) and the row time; Wm becomes W_eff = Rd W
        if (RS) {
            tau = rs.row_time[id];
            rolling_shutter_rotation(tau, rs.motion + 3, Rd);
#pragma unroll
            for (int k = 0; k < 9; ++k) Wo[k] = Wm[k];
#pragma unroll
            for (int r = 0; r < 3; ++r)
#pragma unroll
                for (int c = 0; c < 3; ++c) Wm[3 * r + c] = (Rd[3 * r] * Wo[c] + Rd[3 * r + 1] * Wo[3 + c]) + Rd[3 * r + 2] * Wo[6 + c];
        }

        // d uv / d xyz (GP3D:132-159): full-K projection Jacobian times W
        const float iz = 1.0f / pcz, iz2 = iz * iz;
        float dj[6] = {Kc[0] * iz, Kc[1] * iz, (-Kc[0] * pcx - Kc[1] * pcy) * iz2,
                       Kc[3] * iz, Kc[4] * iz, (-Kc[3] * pcx - Kc[4] * pcy) * iz2};
        float Jl[6];  // LENS: diag(fx, fy) D P, the J of Sigma' below
        float Mk[4] = {Kc[0], Kc[1], Kc[3], Kc[4]};  // DEFOCUS: M = K[:2,:2] (K[:2,:2] D with LENS)
        float ox, oy, D[4];  // LENS: (xd, yd) - (xn, yn) and D = d(xd, yd)/d(xn, yn) at the point
        if (LENS) {
            if (lens.model == GSB_LENS_FISHEYE) lens_distort<GSB_LENS_FISHEYE>(lens.k, pcx * iz, pcy * iz, ox, oy, D);
            else lens_distort<GSB_LENS_OPENCV>(lens.k, pcx * iz, pcy * iz, ox, oy, D);
            // K[:2,:2] D P: the pinhole expression with K[:2,:2] replaced by K[:2,:2] D (exactly K[:2,:2] for D = I)
            const float A0 = Kc[0] * D[0] + Kc[1] * D[2], A1 = Kc[0] * D[1] + Kc[1] * D[3];
            const float A3 = Kc[3] * D[0] + Kc[4] * D[2], A4 = Kc[3] * D[1] + Kc[4] * D[3];
            Mk[0] = A0; Mk[1] = A1; Mk[2] = A3; Mk[3] = A4;
            dj[0] = A0 * iz; dj[1] = A1 * iz; dj[2] = (-A0 * pcx - A1 * pcy) * iz2;
            dj[3] = A3 * iz; dj[4] = A4 * iz; dj[5] = (-A3 * pcx - A4 * pcy) * iz2;
            const float F0 = Kc[0] * D[0], F1 = Kc[0] * D[1], F3 = Kc[4] * D[2], F4 = Kc[4] * D[3];  // likewise
            Jl[0] = F0 * iz; Jl[1] = F1 * iz; Jl[2] = -(F0 * pcx + F1 * pcy) * iz2;
            Jl[3] = F3 * iz; Jl[4] = F4 * iz; Jl[5] = -(F3 * pcx + F4 * pcy) * iz2;
        }
        float eq_r = 1.0f;  // EQUI: the ray distance r
        if (EQUI) {  // d uv / d pc = J of the panorama
            const float pcv[3] = {pcx, pcy, pcz};
            const float rho = sqrtf(pcx * pcx + pcz * pcz);
            eq_r = sqrtf(rho * rho + pcy * pcy);
            equirect_jacobian(Kc[0], Kc[4], pcv, rho, eq_r, dj);
        }
        if (ORTHO) {  // d uv / d pc = K[:2,:2] [I 0]
            dj[0] = Kc[0]; dj[1] = Kc[1]; dj[2] = 0.0f;
            dj[3] = Kc[3]; dj[4] = Kc[4]; dj[5] = 0.0f;
        }
        float gx[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float d0 = dj[0] * Wm[c] + dj[1] * Wm[3 + c] + dj[2] * Wm[6 + c];
            const float d1 = dj[3] * Wm[c] + dj[4] * Wm[3 + c] + dj[5] * Wm[6 + c];
            gx[c] = a0.x * d0 + a0.y * d1;
            if (DEPTH && !EQUI) gx[c] += a2.w * Wm[6 + c];
            if (DEPTH && EQUI) gx[c] += a2.w * (((pcx * Wm[c] + pcy * Wm[3 + c]) + pcz * Wm[6 + c]) / eq_r);  // dr/dpc = pc / r
        }
        // Sigma' = U Sigma U^T, U = J W with J from fx, fy only (GP3D:65-87, 237-331)
        const float fx = Kc[0], fy = Kc[4];
        float J[6] = {fx * iz, 0.0f, -(fx * pcx) * iz2, 0.0f, fy * iz, -(fy * pcy) * iz2};
        if (LENS) {
#pragma unroll
            for (int k = 0; k < 6; ++k) J[k] = Jl[k];
        }
        if (EQUI || ORTHO) {
#pragma unroll
            for (int k = 0; k < 6; ++k) J[k] = dj[k];
        }
        float U[6];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            U[c] = J[0] * Wm[c] + J[1] * Wm[3 + c] + J[2] * Wm[6 + c];
            U[3 + c] = J[3] * Wm[c] + J[4] * Wm[3 + c] + J[5] * Wm[6 + c];
        }
        float g00 = 0.5f * a0.z, g01 = 0.5f * a0.w, g11 = 0.5f * a1.x;  // UT:345's 1/2, see the blend loop
        const bool moving = BLUR && motion_blur_on(blur.motion);
        const bool defocused = DEFOCUS && defocus.aperture != 0.0f;
        if (moving || defocused) {
            // Sigma' = (U M)(U M)^T, M = R(q) diag(exp(s)) (the rows of R and exp(s) as below)
            const float bx = qv.x, by = qv.y, bz = qv.z, bw = qv.w;
            const float Rb[9] = {1 - 2 * (by * by + bz * bz), 2 * (bx * by - bw * bz), 2 * (bx * bz + bw * by),
                                 2 * (bx * by + bw * bz), 1 - 2 * (bx * bx + bz * bz), 2 * (by * bz - bw * bx),
                                 2 * (bx * bz - bw * by), 2 * (by * bz + bw * bx), 1 - 2 * (bx * bx + by * by)};
            const float eb[3] = {expf(sv.x), expf(sv.y), expf(sv.z)};
            float UM[6];
#pragma unroll
            for (int a = 0; a < 2; ++a)
#pragma unroll
                for (int j = 0; j < 3; ++j)
                    UM[a * 3 + j] = (U[a * 3] * Rb[j] + U[a * 3 + 1] * Rb[3 + j] + U[a * 3 + 2] * Rb[6 + j]) * eb[j];
            const float s00 = UM[0] * UM[0] + UM[1] * UM[1] + UM[2] * UM[2];
            const float s01 = UM[0] * UM[3] + UM[1] * UM[4] + UM[2] * UM[5];
            const float s11 = UM[3] * UM[3] + UM[4] * UM[4] + UM[5] * UM[5];
            const float pcv[3] = {pcx, pcy, pcz};
            float d0 = 0.0f, d1 = 0.0f, gd0, gd1;
            if (moving) motion_blur_velocity(dj, pcv, blur.motion, d0, d1);
            const float one_minus_o = 1.0f - __ldg(p.records + 3 * (size_t)o + 1).z;
            const float g_alpha = one_minus_o != 0.0f ? a2.x / one_minus_o : 0.0f;
            if (!defocused) {
                motion_blur_grad(s00, s01, s11, d0, d1, g_alpha, g00, g01, g11, gd0, gd1);
                if (BGRAD) {  // g = Jp^T dL/dd: dL/dv = g, dL/dw = pc x g
                    const float q0 = dj[0] * gd0 + dj[3] * gd1, q1 = dj[1] * gd0 + dj[4] * gd1, q2 = dj[2] * gd0 + dj[5] * gd1;
                    mv[0] = q0; mv[1] = q1; mv[2] = q2;
                    mv[3] = pcy * q2 - pcz * q1;
                    mv[4] = pcz * q0 - pcx * q2;
                    mv[5] = pcx * q1 - pcy * q0;
                }
            } else {  // B = d d^T / 12 (zero without motion) + beta M M^T
                const float P00 = Mk[0] * Mk[0] + Mk[1] * Mk[1], P01 = Mk[0] * Mk[2] + Mk[1] * Mk[3],
                            P11 = Mk[2] * Mk[2] + Mk[3] * Mk[3];
                const float beta = defocus_variance(defocus, pcz);
                const float b00 = (d0 * d0) / 12.0f + beta * P00, b01 = (d0 * d1) / 12.0f + beta * P01,
                            b11 = (d1 * d1) / 12.0f + beta * P11;
                float h00, h01, h11;
                blur_cov_grad(s00, s01, s11, b00, b01, b11, g_alpha, g00, g01, g11, h00, h01, h11);
                if (DGRAD) {
                    const float gbeta = h00 * P00 + 2.0f * (h01 * P01) + h11 * P11;
                    const float e = defocus.inverse_focus - 1.0f / pcz, a = defocus.aperture;
                    mv[0] = gbeta * (a * (e * e)) / 8.0f;
                    mv[1] = gbeta * ((a * a) * e) / 8.0f;
                }
            }
        }
        // V = U^T G U  (dL/dSigma with the (g00,g01,g01,g11) weighting of GPCR:716-721)
        float V[9];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float t0 = g00 * U[k] + g01 * U[3 + k];
            const float t1 = g01 * U[k] + g11 * U[3 + k];
#pragma unroll
            for (int l = 0; l < 3; ++l) V[k * 3 + l] = t0 * U[l] + t1 * U[3 + l];
        }
        // R(q) (GP3D:30-48), M = R S
        const float qx = qv.x, qy = qv.y, qz = qv.z, qw = qv.w;
        float R[9];
        R[0] = 1 - 2 * (qy * qy + qz * qz); R[1] = 2 * (qx * qy - qw * qz); R[2] = 2 * (qx * qz + qw * qy);
        R[3] = 2 * (qx * qy + qw * qz); R[4] = 1 - 2 * (qx * qx + qz * qz); R[5] = 2 * (qy * qz - qw * qx);
        R[6] = 2 * (qx * qz - qw * qy); R[7] = 2 * (qy * qz + qw * qx); R[8] = 1 - 2 * (qx * qx + qy * qy);
        float es[3] = {expf(sv.x), expf(sv.y), expf(sv.z)};  // FILTER: s^
        float fr[3] = {1.0f, 1.0f, 1.0f}, fcomp[3] = {0.0f, 0.0f, 0.0f};  // FILTER: e / e^ and G_a sigma^2 / e^
        bool filtered = false;  // FILTER: sigma > 0 (sigma = 0 leaves the row's gradient exactly as unfiltered)
        if (FILTER) {
            const float sg = fmaxf(filter3d[id], 0.0f);  // NaN -> 0, as the forward
            const float s2 = sg * sg;
            filtered = s2 > 0.0f;
            if (filtered) {
                const float one_minus_o = 1.0f - __ldg(p.records + 3 * (size_t)o + 1).z;
                const float g_alpha = one_minus_o != 0.0f ? a2.x / one_minus_o : 0.0f;
#pragma unroll
                for (int j = 0; j < 3; ++j) {
                    const float e = es[j] * es[j], eh = e + s2;
                    fr[j] = e / eh;
                    fcomp[j] = g_alpha * (s2 / eh);
                    es[j] = sqrtf(eh);
                }
            }
        }
        // dL/dM = (V + V^T) M,  M_ij = R_ij es_j
        float dM[9];
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int b = 0; b < 3; ++b) {
                float acc = 0.0f;
#pragma unroll
                for (int l = 0; l < 3; ++l) acc += (V[a * 3 + l] + V[l * 3 + a]) * (R[l * 3 + b] * es[b]);
                dM[a * 3 + b] = acc;
            }
        // d/ds_j = sum_i dM_ij R_ij es_j
        float gs[3];
#pragma unroll
        for (int j = 0; j < 3; ++j) gs[j] = (dM[j] * R[j] + dM[3 + j] * R[3 + j] + dM[6 + j] * R[6 + j]) * es[j];
        if (FILTER && filtered) {
#pragma unroll
            for (int j = 0; j < 3; ++j) gs[j] = gs[j] * fr[j] + fcomp[j];
        }
        // d/dq = sum_ij dM_ij es_j dR_ij/dq  (table GP3D:316-329)
        const float sx = es[0], sy = es[1], sz = es[2];
        float gq[4];
        gq[0] = dM[1] * (2 * sy * qy) + dM[2] * (2 * sz * qz) + dM[3] * (2 * sx * qy) + dM[4] * (-4 * sy * qx) +
                dM[5] * (-2 * sz * qw) + dM[6] * (2 * sx * qz) + dM[7] * (2 * sy * qw) + dM[8] * (-4 * sz * qx);
        gq[1] = dM[0] * (-4 * sx * qy) + dM[1] * (2 * sy * qx) + dM[2] * (2 * sz * qw) + dM[3] * (2 * sx * qx) +
                dM[5] * (2 * sz * qz) + dM[6] * (-2 * sx * qw) + dM[7] * (2 * sy * qz) + dM[8] * (-4 * sz * qy);
        gq[2] = dM[0] * (-4 * sx * qz) + dM[1] * (-2 * sy * qw) + dM[2] * (2 * sz * qx) + dM[3] * (2 * sx * qw) +
                dM[4] * (-4 * sy * qz) + dM[5] * (2 * sz * qy) + dM[6] * (2 * sx * qx) + dM[7] * (2 * sy * qy);
        gq[3] = dM[1] * (-2 * sy * qz) + dM[2] * (2 * sz * qy) + dM[3] * (2 * sx * qz) + dM[5] * (-2 * sz * qx) +
                dM[6] * (-2 * sx * qy) + dM[7] * (2 * sy * qx);
        // sigmoid'(.) from the stored colour: c (1 - c)  (UT:356-359)
        const float gcol[3] = {a1.y * (r2.x * (1.0f - r2.x)), a1.z * (r2.y * (1.0f - r2.y)),
                               a1.w * (r2.z * (1.0f - r2.z))};
        if (POSE) {
            // pc = W xyz + tw.  gp = dL/dpc through uv (and z with DEPTH): dL/dW += gp xyz^T, dL/dtw += gp.
            // Sigma' = U Sigma U^T with U = J W (J detached): dL/dU = 2 G U Sigma, dL/dW += J^T (2 G U Sigma)
            float gp[3];
#pragma unroll
            for (int r = 0; r < 3; ++r) gp[r] = dj[r] * a0.x + dj[3 + r] * a0.y;
            if (DEPTH) gp[2] += a2.w;
            float B0[3], B1[3];
            weighted_u_sigma(U, R, es, g00, g01, g11, B0, B1);
            const float xw[3] = {x, y, z};
#pragma unroll
            for (int c = 0; c < 3; ++c) {  // J = [J0 0 J2; 0 J4 J5]; ORTHO: J = [J0 J1 0; J3 J4 0]
                if (ORTHO) {
                    pv[c] = gp[0] * xw[c] + 2.0f * (J[0] * B0[c] + J[3] * B1[c]);
                    pv[3 + c] = gp[1] * xw[c] + 2.0f * (J[1] * B0[c] + J[4] * B1[c]);
                    pv[6 + c] = gp[2] * xw[c];
                } else if (LENS) {  // J = diag(fx, fy) D P: all six entries
                    pv[c] = gp[0] * xw[c] + 2.0f * (J[0] * B0[c] + J[3] * B1[c]);
                    pv[3 + c] = gp[1] * xw[c] + 2.0f * (J[1] * B0[c] + J[4] * B1[c]);
                    pv[6 + c] = gp[2] * xw[c] + 2.0f * (J[2] * B0[c] + J[5] * B1[c]);
                } else {
                    pv[c] = gp[0] * xw[c] + 2.0f * (J[0] * B0[c]);
                    pv[3 + c] = gp[1] * xw[c] + 2.0f * (J[4] * B1[c]);
                    pv[6 + c] = gp[2] * xw[c] + 2.0f * (J[2] * B0[c] + J[5] * B1[c]);
                }
                pv[9 + c] = gp[c];
            }
            pose_obj = ob;
        }
        if (INTR) {
            // uv = (K pc)[:2] / z: dL/dK[r][c] += guv_r pc_c / z.  Sigma' through J = [fx/z 0 -fx x/z^2; 0 fy/z -fy y/z^2]
            // (pc detached in J): dL/dfx += 2 sum_c B0[c] (W[0][c]/z - x W[2][c]/z^2), dL/dfy likewise with B1 and row 1
            float B0[3], B1[3];
            weighted_u_sigma(U, R, es, g00, g01, g11, B0, B1);
            if (ORTHO) {
                // uv = K[:2] (x, y, 1): dL/dK[r][c] += guv_r (x, y, 1)_c.  Sigma' through J = K[:2,:2] [I 0]:
                // dL/dK[r][c] += 2 sum_j B_r[j] W[c][j] for c in {0, 1}
                float s00 = 0.0f, s01 = 0.0f, s10 = 0.0f, s11 = 0.0f;
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    s00 += B0[c] * Wm[c];
                    s01 += B0[c] * Wm[3 + c];
                    s10 += B1[c] * Wm[c];
                    s11 += B1[c] * Wm[3 + c];
                }
                iv[0] = a0.x * pcx + 2.0f * s00;
                iv[1] = a0.x * pcy + 2.0f * s01;
                iv[2] = a0.x;
                iv[3] = a0.y * pcx + 2.0f * s10;
                iv[4] = a0.y * pcy + 2.0f * s11;
                iv[5] = a0.y;
            } else if (LENS) {
                // uv = K[:2] (xd, yd, 1): dL/dK[r][c] += guv_r (xd, yd, 1)_c.  Sigma' through J = diag(fx, fy) D P:
                // dL/dfx += 2 sum_c B0[c] (D P W)[0][c], dL/dfy likewise with B1 and row 1 (D = I: the pinhole's)
                const float xd = pcx * iz + ox, yd = pcy * iz + oy;
                const float P0[3] = {D[0] * iz, D[1] * iz, -(D[0] * pcx + D[1] * pcy) * iz2};  // rows of D P
                const float P1[3] = {D[2] * iz, D[3] * iz, -(D[2] * pcx + D[3] * pcy) * iz2};
                float sx0 = 0.0f, sy1 = 0.0f;
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    sx0 += B0[c] * ((P0[0] * Wm[c] + P0[1] * Wm[3 + c]) + P0[2] * Wm[6 + c]);
                    sy1 += B1[c] * ((P1[0] * Wm[c] + P1[1] * Wm[3 + c]) + P1[2] * Wm[6 + c]);
                }
                iv[0] = a0.x * xd + 2.0f * sx0;
                iv[1] = a0.x * yd;
                iv[2] = a0.x;
                iv[3] = a0.y * xd;
                iv[4] = a0.y * yd + 2.0f * sy1;
                iv[5] = a0.y;
            } else {
            const float ux = pcx * iz, uy = pcy * iz;
            float sx0 = 0.0f, sy1 = 0.0f;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                sx0 += B0[c] * (Wm[c] * iz - (pcx * Wm[6 + c]) * iz2);
                sy1 += B1[c] * (Wm[3 + c] * iz - (pcy * Wm[6 + c]) * iz2);
            }
            iv[0] = a0.x * ux + 2.0f * sx0;
            iv[1] = a0.x * uy;
            iv[2] = a0.x;
            iv[3] = a0.y * ux;
            iv[4] = a0.y * uy + 2.0f * sy1;
            iv[5] = a0.y;
            }
        }
        if (LGRAD) {
            // position: dL/d(xd, yd) = K[:2,:2]^T guv.  Sigma' through J = diag(fx, fy) D P (pc detached, D differentiated in k
            // alone): dL/dJ = 2 [B0; B1] W^T, dL/dD = diag(fx, fy) dL/dJ P^T
            float B0[3], B1[3];
            weighted_u_sigma(U, R, es, g00, g01, g11, B0, B1);
            float h0[3], h1[3];  // [B0; B1] W^T
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                h0[j] = B0[0] * Wm[3 * j] + B0[1] * Wm[3 * j + 1] + B0[2] * Wm[3 * j + 2];
                h1[j] = B1[0] * Wm[3 * j] + B1[1] * Wm[3 * j + 1] + B1[2] * Wm[3 * j + 2];
            }
            const float gxd = Kc[0] * a0.x + Kc[3] * a0.y, gyd = Kc[1] * a0.x + Kc[4] * a0.y;
            const float w00 = 2.0f * fx * (h0[0] * iz - (h0[2] * pcx) * iz2), w01 = 2.0f * fx * (h0[1] * iz - (h0[2] * pcy) * iz2);
            const float w10 = 2.0f * fy * (h1[0] * iz - (h1[2] * pcx) * iz2), w11 = 2.0f * fy * (h1[1] * iz - (h1[2] * pcy) * iz2);
            if (lens.model == GSB_LENS_FISHEYE)
                lens_coefficient_grad<GSB_LENS_FISHEYE>(pcx * iz, pcy * iz, gxd, gyd, w00, w01 + w10, w11, lv);
            else lens_coefficient_grad<GSB_LENS_OPENCV>(pcx * iz, pcy * iz, gxd, gyd, w00, w01 + w10, w11, lv);
        }
        if (MGRAD) {
            // gp = dL/dpc(tau) through uv (and z with DEPTH); Sigma' = U Sigma U^T with U = J Rd W: dL/dU = 2 [B0; B1]
            float gp[3];
#pragma unroll
            for (int r = 0; r < 3; ++r) gp[r] = dj[r] * a0.x + dj[3 + r] * a0.y;
            if (DEPTH) gp[2] += a2.w;
            float B0[3], B1[3];
            weighted_u_sigma(U, R, es, g00, g01, g11, B0, B1);
            const float pc0[3] = {((Wo[0] * x + Wo[1] * y) + Wo[2] * z) + pb->T[3],
                                  ((Wo[3] * x + Wo[4] * y) + Wo[5] * z) + pb->T[7],
                                  ((Wo[6] * x + Wo[7] * y) + Wo[8] * z) + pb->T[11]};
            rolling_shutter_grad(tau, rs.motion + 3, Rd, pc0, gp, J, B0, B1, Wo, mv);
        }
        if (p.ctl_num_in_camera != nullptr && !(p.skip_flag != nullptr && *p.skip_flag != 0)) {
            // GaussianPointAdaptiveController.update (:130-143) for this in-camera point: ids are unique, one thread per row,
            // so plain read-modify-writes.  a2.y = sum |d/duv| over pixels, a2.z = number of affected pixels (exact in f32)
            const int npix = __float2int_rn(a2.z);
            p.ctl_num_in_camera[id] += 1;
            p.ctl_num_pixels[id] += npix;
            p.ctl_vs_grad[id] += a2.y;
            float avg = a2.y / (float)npix;  // 0/0 -> NaN -> 0; x/0 stays inf like the reference
            if (avg != avg) avg = 0.0f;
            p.ctl_vs_grad_avg[id] += avg;
            p.ctl_pos_grad[3 * id] += gx[0];
            p.ctl_pos_grad[3 * id + 1] += gx[1];
            p.ctl_pos_grad[3 * id + 2] += gx[2];
            p.ctl_pos_grad_norm[id] += sqrtf(gx[0] * gx[0] + gx[1] * gx[1] + gx[2] * gx[2]);
        }
        if (COMPACT) {
            float4 *gc = reinterpret_cast<float4 *>(my_feat);
            gc[0] = make_float4(gx[0], gx[1], gx[2], gq[0] * p.q_f);
            gc[1] = make_float4(gq[1] * p.q_f, gq[2] * p.q_f, gq[3] * p.q_f, gs[0] * p.s_f);
            gc[2] = make_float4(gs[1] * p.s_f, gs[2] * p.s_f, a2.x * p.a_f, 0.0f);
            gc[3] = make_float4(gcol[0], gcol[1], gcol[2], 0.0f);
        } else {
        // SH basis along xyz - camera centre (GPCR:731-732, 749; SH:10-32)
        float sh[16];
        if (ORTHO) sh_basis(Wm[6], Wm[7], Wm[8], sh);  // the camera's forward axis, as the forward
        else sh_basis(x - p.t_pc_cam[3 * ob], y - p.t_pc_cam[3 * ob + 1], z - p.t_pc_cam[3 * ob + 2], sh);

        my_xyz[0] = gx[0]; my_xyz[1] = gx[1]; my_xyz[2] = gx[2];
        float4 *gf = reinterpret_cast<float4 *>(my_feat);
        gf[0] = make_float4(gq[0] * p.q_f, gq[1] * p.q_f, gq[2] * p.q_f, gq[3] * p.q_f);
        gf[1] = make_float4(gs[0] * p.s_f, gs[1] * p.s_f, gs[2] * p.s_f, a2.x * p.a_f);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
            float o16[16];
#pragma unroll
            for (int k = 0; k < 16; ++k) {
                const float factor = k == 0 ? p.c_f : p.h_f;
                o16[k] = k < p.first_cleared ? gcol[ch] * sh[k] * factor : 0.0f;
            }
#pragma unroll
            for (int k4 = 0; k4 < 4; ++k4)
                gf[2 + 4 * ch + k4] = make_float4(o16[4 * k4], o16[4 * k4 + 1], o16[4 * k4 + 2], o16[4 * k4 + 3]);
        }
        }
      }
      if (POSE) {
          // one pass per object present in the warp (points of several objects may share a warp), lowest lane's first
          unsigned int todo = __ballot_sync(0xffffffffu, pose_obj >= 0);
          while (todo) {
              const int cur = __shfl_sync(0xffffffffu, pose_obj, __ffs(todo) - 1);
              const bool mine = pose_obj == cur;
              todo &= ~__ballot_sync(0xffffffffu, mine);
#pragma unroll
              for (int k = 0; k < POSE_VALUES; ++k) {
                  float v = mine ? pv[k] : 0.0f;
#pragma unroll
                  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
                  if (lane == 0) my_pose[cur * POSE_VALUES + k] += v;
              }
          }
      }
      if (INTR) {
#pragma unroll
          for (int k = 0; k < INTR_VALUES; ++k) {
              float v = iv[k];
#pragma unroll
              for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
              if (lane == 0) my_intr[k] += v;
          }
      }
      if (LGRAD) {
#pragma unroll
          for (int k = 0; k < LENS_GRAD_VALUES; ++k) {
              float v = lv[k];
#pragma unroll
              for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
              if (lane == 0) my_lgrad[k] += v;
          }
      }
      if (CAM6) {
#pragma unroll
          for (int k = 0; k < RS_GRAD_VALUES; ++k) {
              float v = mv[k];
#pragma unroll
              for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
              if (lane == 0) my_mgrad[k] += v;
          }
      }
      __syncwarp();
      const long long rows = p.N - base < 32 ? p.N - base : 32;
      if (COMPACT) {
          // 32 rows -> 3 x 512 B of summable columns, 3 x 128 B of per-view colour gradients
          float4 *const out_s = reinterpret_cast<float4 *>(p.grad_sum_compact + 12 * (size_t)base);
          float *const out_c = p.grad_color_compact + 3 * (size_t)base;
#pragma unroll
          for (int it = 0; it < 3; ++it) {
              const int f = it * 32 + lane;
              const int row = f / 3, c = f - row * 3;
              if (row < rows) {
                  out_s[f] = *reinterpret_cast<const float4 *>(&s_feat[warp][row * ROW + 4 * c]);
                  out_c[f] = s_feat[warp][row * ROW + 12 + c];
              }
          }
      } else {
      // stream the warp's 32 rows out: 14 x 512 B of feature gradients, 3 x 128 B of position gradients
      float4 *const out_f = reinterpret_cast<float4 *>(p.grad_feat + (size_t)GSB_FEATURE_DIM * base);
#pragma unroll
      for (int it = 0; it < GSB_FEATURE_DIM / 4; ++it) {
          const int f = it * 32 + lane;           // float4 index inside the piece
          const int row = f / (GSB_FEATURE_DIM / 4), c4 = f - row * (GSB_FEATURE_DIM / 4);
          if (row < rows) out_f[f] = *reinterpret_cast<const float4 *>(&s_feat[warp][row * ROW + 4 * c4]);
      }
      float *const out_x = p.grad_xyz + 3 * (size_t)base;
#pragma unroll
      for (int it = 0; it < 3; ++it) {
          const int f = it * 32 + lane;
          if (f < 3 * rows) out_x[f] = s_xyz[warp][f];
      }
      }
      __syncwarp();
    }
    if (POSE) {
        __syncthreads();
        float *const out = pose_partials + (size_t)blockIdx.x * num_objects * POSE_VALUES;
        for (int k = threadIdx.x; k < num_objects * POSE_VALUES; k += blockDim.x) {
            float s = s_pose[k];
            for (int w = 1; w < GSB_POINTS_THREADS / 32; ++w) s += s_pose[w * num_objects * POSE_VALUES + k];
            out[k] = s;
        }
    }
    if (INTR) {
        __syncthreads();
        if (threadIdx.x < INTR_VALUES) {
            float s = s_intr[threadIdx.x];
            for (int w = 1; w < GSB_POINTS_THREADS / 32; ++w) s += s_intr[w * INTR_VALUES + threadIdx.x];
            intr_partials[(size_t)blockIdx.x * INTR_VALUES + threadIdx.x] = s;
        }
    }
    if (LGRAD) {
        __syncthreads();
        if (threadIdx.x < LENS_GRAD_VALUES) {
            float s = s_lgrad[threadIdx.x];
            for (int w = 1; w < GSB_POINTS_THREADS / 32; ++w) s += s_lgrad[w * LENS_GRAD_VALUES + threadIdx.x];
            lgrad_partials[(size_t)blockIdx.x * LENS_GRAD_VALUES + threadIdx.x] = s;
        }
    }
    if (CAM6) {
        __syncthreads();
        if (threadIdx.x < RS_GRAD_VALUES) {
            float s = s_mgrad[threadIdx.x];
            for (int w = 1; w < GSB_POINTS_THREADS / 32; ++w) s += s_mgrad[w * RS_GRAD_VALUES + threadIdx.x];
            mgrad_partials[(size_t)blockIdx.x * RS_GRAD_VALUES + threadIdx.x] = s;
        }
    }
}

template <bool COMPACT, bool DEPTH = false>
__global__ void __launch_bounds__(GSB_POINTS_THREADS, 6)  // 6 x 33 KB of staging per SM
backward_points_kernel(const PointsBwdParams p) {
    backward_points_body<COMPACT, DEPTH, false>(p, nullptr, nullptr, 0);
}

// The parameter block of the POSE instantiations: the default kernels keep PointsBwdParams as it is.
struct PointsBwdPoseParams : PointsBwdParams {
    float *pose_partials;  // (grid, num_objects, 12)
    int num_objects;       // <= GSB_POSE_MAX_OBJECTS
};

template <bool DEPTH>
__global__ void __launch_bounds__(GSB_POINTS_THREADS, 5)  // + 12 KB of per-warp pose rows
backward_points_pose_kernel(const PointsBwdPoseParams p) {
    __shared__ float s_pose[(GSB_POINTS_THREADS / 32) * GSB_POSE_MAX_OBJECTS * POSE_VALUES];
    backward_points_body<false, DEPTH, true>(p, s_pose, p.pose_partials, p.num_objects);
}

// The parameter block of the LENS instantiations: the default kernels keep PointsBwdParams as it is.
struct PointsBwdLensParams : PointsBwdParams {
    LensParams lens;
};

template <bool DEPTH>
__global__ void __launch_bounds__(GSB_POINTS_THREADS, 5)  // at 6 CTAs per SM the lens Jacobians spill 4-8 bytes
backward_points_lens_kernel(const PointsBwdLensParams p) {
    backward_points_body<false, DEPTH, false, false, true>(p, nullptr, nullptr, 0, nullptr, nullptr, p.lens);
}

// The parameter block of the LGRAD instantiations.
struct PointsBwdLensGradParams : PointsBwdLensParams {
    float *lens_partials;  // (grid, 5)
};

template <bool DEPTH>
__global__ void __launch_bounds__(GSB_POINTS_THREADS, 4)  // 5 values live across the SH epilogue: at 5 CTAs per SM it spills
backward_points_lens_grad_kernel(const PointsBwdLensGradParams p) {
    __shared__ float s_lgrad[(GSB_POINTS_THREADS / 32) * LENS_GRAD_VALUES];
    backward_points_body<false, DEPTH, false, false, true, true>(p, nullptr, nullptr, 0, nullptr, nullptr, p.lens, s_lgrad,
                                                                 p.lens_partials);
}

template <bool DEPTH>
__global__ void __launch_bounds__(GSB_POINTS_THREADS, 6)
backward_points_equirect_kernel(const PointsBwdParams p) {
    backward_points_body<false, DEPTH, false, false, false, false, false, false, false, false, false, false, false, true>(
        p, nullptr, nullptr, 0);
}

// One CTA: adds the `blocks` partial rows in a fixed order (strided per thread, then a fixed shared-memory tree) and writes
// the 5 coefficient gradients (the unused fifth of a fisheye lens is a sum of zeros).  Zeros when blocks == 0.
constexpr int LENS_GRAD_FINISH_THREADS = 128;
__global__ void __launch_bounds__(LENS_GRAD_FINISH_THREADS)
lens_grad_finish_kernel(const float *__restrict__ partials, int blocks, float *__restrict__ grad_coefficients) {
    __shared__ float s_sum[LENS_GRAD_FINISH_THREADS][LENS_GRAD_VALUES + 1];
    const int tid = threadIdx.x;
    float acc[LENS_GRAD_VALUES];
#pragma unroll
    for (int k = 0; k < LENS_GRAD_VALUES; ++k) acc[k] = 0.0f;
    for (int b = tid; b < blocks; b += LENS_GRAD_FINISH_THREADS) {
#pragma unroll
        for (int k = 0; k < LENS_GRAD_VALUES; ++k) acc[k] += partials[(size_t)b * LENS_GRAD_VALUES + k];
    }
#pragma unroll
    for (int k = 0; k < LENS_GRAD_VALUES; ++k) s_sum[tid][k] = acc[k];
    __syncthreads();
    for (int h = LENS_GRAD_FINISH_THREADS / 2; h > 0; h >>= 1) {
        if (tid < h)
#pragma unroll
            for (int k = 0; k < LENS_GRAD_VALUES; ++k) s_sum[tid][k] += s_sum[tid + h][k];
        __syncthreads();
    }
    if (tid < LENS_GRAD_VALUES) grad_coefficients[tid] = s_sum[0][tid];
}

// The parameter block of the rolling-shutter instantiations (LENS = false ignores `lens`).
struct PointsBwdRsParams : PointsBwdLensParams {
    RsParams rs;
    float *rs_partials;  // MGRAD: (grid, 6)
};

template <bool DEPTH, bool LENS, bool MGRAD>
__global__ void __launch_bounds__(GSB_POINTS_THREADS, MGRAD ? 3 : 5)  // MGRAD: at 4 CTAs per SM the 6 values spill 4 bytes
backward_points_rs_kernel(const PointsBwdRsParams p) {
    __shared__ float s_mgrad[MGRAD ? (GSB_POINTS_THREADS / 32) * RS_GRAD_VALUES : 1];
    backward_points_body<false, DEPTH, false, false, LENS, false, true, MGRAD>(p, nullptr, nullptr, 0, nullptr, nullptr, p.lens,
                                                                              nullptr, nullptr, p.rs, s_mgrad, p.rs_partials);
}

// The parameter blocks of the FILTER instantiations (LENS = false ignores `lens`).
struct PointsBwdFilterParams : PointsBwdLensParams {
    const float *filter3d;
};
struct PointsBwdRsFilterParams : PointsBwdRsParams {
    const float *filter3d;
};

template <bool DEPTH, bool LENS>
__global__ void __launch_bounds__(GSB_POINTS_THREADS, LENS ? 5 : 6)
backward_points_filter_kernel(const PointsBwdFilterParams p) {
    backward_points_body<false, DEPTH, false, false, LENS, false, false, false, true>(
        p, nullptr, nullptr, 0, nullptr, nullptr, p.lens, nullptr, nullptr, RsParams(), nullptr, nullptr, p.filter3d);
}

template <bool DEPTH, bool LENS>
__global__ void __launch_bounds__(GSB_POINTS_THREADS, 5)
backward_points_rs_filter_kernel(const PointsBwdRsFilterParams p) {
    backward_points_body<false, DEPTH, false, false, LENS, false, true, false, true>(
        p, nullptr, nullptr, 0, nullptr, nullptr, p.lens, nullptr, nullptr, p.rs, nullptr, nullptr, p.filter3d);
}

// The parameter block of the BLUR instantiations (LENS = false ignores `lens`, RS = false ignores `rs`; rs_partials: the
// BGRAD or DGRAD rows; DEFOCUS = false ignores `defocus`).
struct PointsBwdBlurParams : PointsBwdRsParams {
    BlurParams blur;
    DefocusParams defocus;
};

template <bool DEPTH, bool LENS, bool RS, bool BGRAD, bool DEFOCUS = false, bool DGRAD = false>
__global__ void __launch_bounds__(GSB_POINTS_THREADS, BGRAD || DGRAD ? 3 : 5)
backward_points_blur_kernel(const PointsBwdBlurParams p) {
    __shared__ float s_mgrad[BGRAD || DGRAD ? (GSB_POINTS_THREADS / 32) * RS_GRAD_VALUES : 1];
    backward_points_body<false, DEPTH, false, false, LENS, false, RS, false, false, true, BGRAD, DEFOCUS, DGRAD>(
        p, nullptr, nullptr, 0, nullptr, nullptr, p.lens, nullptr, nullptr, p.rs, s_mgrad, p.rs_partials, nullptr, p.blur,
        p.defocus);
}

// One CTA: adds the `blocks` partial rows in a fixed order (strided per thread, then a fixed shared-memory tree) and writes
// the 6 motion gradients (of the rolling shutter or of the exposure).  Zeros when blocks == 0.
constexpr int RS_GRAD_FINISH_THREADS = 128;
__global__ void __launch_bounds__(RS_GRAD_FINISH_THREADS)
rolling_shutter_grad_finish_kernel(const float *__restrict__ partials, int blocks, float *__restrict__ grad_motion) {
    __shared__ float s_sum[RS_GRAD_FINISH_THREADS][RS_GRAD_VALUES + 1];
    const int tid = threadIdx.x;
    float acc[RS_GRAD_VALUES];
#pragma unroll
    for (int k = 0; k < RS_GRAD_VALUES; ++k) acc[k] = 0.0f;
    for (int b = tid; b < blocks; b += RS_GRAD_FINISH_THREADS) {
#pragma unroll
        for (int k = 0; k < RS_GRAD_VALUES; ++k) acc[k] += partials[(size_t)b * RS_GRAD_VALUES + k];
    }
#pragma unroll
    for (int k = 0; k < RS_GRAD_VALUES; ++k) s_sum[tid][k] = acc[k];
    __syncthreads();
    for (int h = RS_GRAD_FINISH_THREADS / 2; h > 0; h >>= 1) {
        if (tid < h)
#pragma unroll
            for (int k = 0; k < RS_GRAD_VALUES; ++k) s_sum[tid][k] += s_sum[tid + h][k];
        __syncthreads();
    }
    if (tid < RS_GRAD_VALUES) grad_motion[tid] = s_sum[0][tid];
}

// R(q) of GP3D:30-48 (xyzw, not normalised) and the gradient of sum_ij G_ij R(q)_ij with respect to q
__device__ __forceinline__ void pose_rot(const float *q, float *R) {
    const float x = q[0], y = q[1], z = q[2], w = q[3];
    R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y - w * z);     R[2] = 2 * (x * z + w * y);
    R[3] = 2 * (x * y + w * z);     R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z - w * x);
    R[6] = 2 * (x * z - w * y);     R[7] = 2 * (y * z + w * x);     R[8] = 1 - 2 * (x * x + y * y);
}
__device__ __forceinline__ void pose_rot_grad(const float *q, const float *G, float *g) {
    const float x = q[0], y = q[1], z = q[2], w = q[3];
    g[0] = 2 * y * (G[1] + G[3]) + 2 * z * (G[2] + G[6]) - 4 * x * (G[4] + G[8]) + 2 * w * (G[7] - G[5]);
    g[1] = 2 * x * (G[1] + G[3]) - 4 * y * (G[0] + G[8]) + 2 * z * (G[5] + G[7]) + 2 * w * (G[2] - G[6]);
    g[2] = 2 * x * (G[2] + G[6]) + 2 * y * (G[5] + G[7]) - 4 * z * (G[0] + G[4]) + 2 * w * (G[3] - G[1]);
    g[3] = 2 * x * (G[7] - G[5]) + 2 * y * (G[2] - G[6]) + 2 * z * (G[3] - G[1]);
}

// One CTA per object: adds the `blocks` partial rows of the object in a fixed order (strided per thread, then a fixed
// shared-memory tree) and takes dL/dW, dL/dtw through pose_kernel's map (preprocess.cu) to dL/dq_pc, dL/dt_pc:
// qi = conj(q_pc), W = R(qi), tw = -R(qn) t_pc with qn = qi / |qi|.  Writes every row, zeros when blocks == 0.
constexpr int POSE_FINISH_THREADS = 128;
__global__ void __launch_bounds__(POSE_FINISH_THREADS)
pose_finish_kernel(const float *__restrict__ partials, int blocks, int num_objects, const float *__restrict__ q_pc,
                   const float *__restrict__ t_pc, float *__restrict__ grad_q, float *__restrict__ grad_t) {
    __shared__ float s_sum[POSE_FINISH_THREADS][POSE_VALUES + 1];
    const int ob = blockIdx.x, tid = threadIdx.x;
    float acc[POSE_VALUES];
#pragma unroll
    for (int k = 0; k < POSE_VALUES; ++k) acc[k] = 0.0f;
    for (int b = tid; b < blocks; b += POSE_FINISH_THREADS) {
        const float *row = partials + ((size_t)b * num_objects + ob) * POSE_VALUES;
#pragma unroll
        for (int k = 0; k < POSE_VALUES; ++k) acc[k] += row[k];
    }
#pragma unroll
    for (int k = 0; k < POSE_VALUES; ++k) s_sum[tid][k] = acc[k];
    __syncthreads();
    for (int h = POSE_FINISH_THREADS / 2; h > 0; h >>= 1) {
        if (tid < h)
#pragma unroll
            for (int k = 0; k < POSE_VALUES; ++k) s_sum[tid][k] += s_sum[tid + h][k];
        __syncthreads();
    }
    if (tid != 0) return;
    const float *gW = s_sum[0], *gtw = s_sum[0] + 9;
    const float qi[4] = {-q_pc[4 * ob], -q_pc[4 * ob + 1], -q_pc[4 * ob + 2], q_pc[4 * ob + 3]};
    const float t[3] = {t_pc[3 * ob], t_pc[3 * ob + 1], t_pc[3 * ob + 2]};
    const float n = sqrtf(((qi[0] * qi[0] + qi[1] * qi[1]) + qi[2] * qi[2]) + qi[3] * qi[3]);
    const float qn[4] = {qi[0] / n, qi[1] / n, qi[2] / n, qi[3] / n};
    float g[4], gn[4], Rn[9], GRn[9];
    pose_rot_grad(qi, gW, g);  // W = R(qi)
    pose_rot(qn, Rn);          // tw = -R(qn) t
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        grad_t[3 * ob + c] = -(Rn[c] * gtw[0] + Rn[3 + c] * gtw[1] + Rn[6 + c] * gtw[2]);
#pragma unroll
        for (int r = 0; r < 3; ++r) GRn[r * 3 + c] = -gtw[r] * t[c];
    }
    pose_rot_grad(qn, GRn, gn);
    const float dot = qn[0] * gn[0] + qn[1] * gn[1] + qn[2] * gn[2] + qn[3] * gn[3];
#pragma unroll
    for (int k = 0; k < 4; ++k) g[k] += (gn[k] - qn[k] * dot) / n;  // d qn / d qi = (I - qn qn^T) / |qi|
    grad_q[4 * ob] = -g[0];  // q_pc = conj(qi)
    grad_q[4 * ob + 1] = -g[1];
    grad_q[4 * ob + 2] = -g[2];
    grad_q[4 * ob + 3] = g[3];
}

// The parameter block of the INTR instantiations (pose_partials / num_objects are read only with POSE).
struct PointsBwdCalibParams : PointsBwdPoseParams {
    float *intr_partials;  // (grid, 6)
};

// Intrinsics alone (POSE = false) or pose and intrinsics in one pass over the scene rows (POSE = true).
template <bool DEPTH, bool POSE>
__global__ void __launch_bounds__(GSB_POINTS_THREADS, POSE ? 4 : 5)  // 6 or 18 values live across the SH epilogue
backward_points_calib_kernel(const PointsBwdCalibParams p) {
    __shared__ float s_pose[POSE ? (GSB_POINTS_THREADS / 32) * GSB_POSE_MAX_OBJECTS * POSE_VALUES : 1];
    __shared__ float s_intr[(GSB_POINTS_THREADS / 32) * INTR_VALUES];
    backward_points_body<false, DEPTH, POSE, true>(p, POSE ? s_pose : nullptr, p.pose_partials, p.num_objects, s_intr,
                                                   p.intr_partials);
}

// The parameter block of the ORTHO instantiations (pose_partials / num_objects read only with POSE, intr_partials only with
// INTR, filter3d only with FILTER).
struct PointsBwdOrthoParams : PointsBwdCalibParams {
    const float *filter3d;
};

template <bool DEPTH, bool POSE, bool INTR, bool FILTER>
__global__ void __launch_bounds__(GSB_POINTS_THREADS, POSE && INTR ? 4 : POSE || INTR ? 5 : 6)  // as the pinhole's kernels
backward_points_ortho_kernel(const PointsBwdOrthoParams p) {
    __shared__ float s_pose[POSE ? (GSB_POINTS_THREADS / 32) * GSB_POSE_MAX_OBJECTS * POSE_VALUES : 1];
    __shared__ float s_intr[INTR ? (GSB_POINTS_THREADS / 32) * INTR_VALUES : 1];
    backward_points_body<false, DEPTH, POSE, INTR, false, false, false, false, FILTER, false, false, false, false, false, true>(
        p, POSE ? s_pose : nullptr, p.pose_partials, p.num_objects, INTR ? s_intr : nullptr, p.intr_partials, LensParams(),
        nullptr, nullptr, RsParams(), nullptr, nullptr, p.filter3d);
}

// The parameter block of the LENS instantiations with camera gradients (pose_partials / num_objects read only with POSE,
// intr_partials only with INTR, lens_partials only with LGRAD).
struct PointsBwdLensCalibParams : PointsBwdCalibParams {
    LensParams lens;
    float *lens_partials;  // (grid, 5)
};

// Pose, intrinsics and coefficient sums through a lens in one pass over the scene rows (POSE or INTR; LGRAD optional).
template <bool DEPTH, bool POSE, bool INTR, bool LGRAD>
__global__ void __launch_bounds__(GSB_POINTS_THREADS, POSE && INTR ? 3 : 4)  // at one CTA per SM more, each of them spills
backward_points_lens_calib_kernel(const PointsBwdLensCalibParams p) {
    static_assert(POSE || INTR, "without camera gradients the lens path is backward_points_lens(_grad)_kernel");
    __shared__ float s_pose[POSE ? (GSB_POINTS_THREADS / 32) * GSB_POSE_MAX_OBJECTS * POSE_VALUES : 1];
    __shared__ float s_intr[INTR ? (GSB_POINTS_THREADS / 32) * INTR_VALUES : 1];
    __shared__ float s_lgrad[LGRAD ? (GSB_POINTS_THREADS / 32) * LENS_GRAD_VALUES : 1];
    backward_points_body<false, DEPTH, POSE, INTR, true, LGRAD>(
        p, POSE ? s_pose : nullptr, p.pose_partials, p.num_objects, INTR ? s_intr : nullptr, p.intr_partials, p.lens,
        LGRAD ? s_lgrad : nullptr, p.lens_partials);
}

// One CTA: adds the `blocks` partial rows in a fixed order (strided per thread, then a fixed shared-memory tree) and
// writes the whole (3,3) dL/dK, row 2 zero (the forward never reads it).  Zeros when blocks == 0.
constexpr int INTR_FINISH_THREADS = 128;
__global__ void __launch_bounds__(INTR_FINISH_THREADS)
intrinsics_finish_kernel(const float *__restrict__ partials, int blocks, float *__restrict__ grad_K) {
    __shared__ float s_sum[INTR_FINISH_THREADS][INTR_VALUES + 1];
    const int tid = threadIdx.x;
    float acc[INTR_VALUES];
#pragma unroll
    for (int k = 0; k < INTR_VALUES; ++k) acc[k] = 0.0f;
    for (int b = tid; b < blocks; b += INTR_FINISH_THREADS) {
#pragma unroll
        for (int k = 0; k < INTR_VALUES; ++k) acc[k] += partials[(size_t)b * INTR_VALUES + k];
    }
#pragma unroll
    for (int k = 0; k < INTR_VALUES; ++k) s_sum[tid][k] = acc[k];
    __syncthreads();
    for (int h = INTR_FINISH_THREADS / 2; h > 0; h >>= 1) {
        if (tid < h)
#pragma unroll
            for (int k = 0; k < INTR_VALUES; ++k) s_sum[tid][k] += s_sum[tid + h][k];
        __syncthreads();
    }
    if (tid < 9) grad_K[tid] = tid < INTR_VALUES ? s_sum[0][tid] : 0.0f;
}

// ------------------------------------------------------------------ view-parallel exchange: rebuild the dense gradients
// After the exchange of the COMPACT rows (parallel.py): grad_sum holds the sum over views of xyz / q / s / logit gradients,
// grad_color_views the per-view colour-argument gradients (3 per row) followed by that view's camera centres.  The SH
// gradient of a view is gcol (x) SH basis(direction from the view's camera centre) * factor (GPCR:749-756, 1105-1125,
// 1167-1182) -- exactly what the dense kernel writes per view -- summed here over the views in rank order (deterministic).
struct ExpandParams {
    long long N;
    int R;
    const float *grad_sum;
    const float *grad_color_views;
    long long view_stride;  // floats between two views' blocks
    const float *xyz;
    const int *obj_id;
    int first_cleared;
    float c_f, h_f;
    float *grad_xyz;
    float *grad_feat;
};

// PART: 0 = everything; 1 = only the 48 SH columns (needs the all-gathered blocks, not the summed rows); 2 = only the summed
// columns xyz / q / s / logit (needs the all-reduced rows, not the blocks).  Parts 1 and 2 write disjoint 32-byte-aligned
// pieces of every row, so part 1 can run -- on another stream -- while the all-reduce is still on the wire (parallel.py).
template <int PART>
__global__ void __launch_bounds__(GSB_POINTS_THREADS, 4)
expand_view_gradients_kernel(const ExpandParams p) {
    __shared__ __align__(16) float s_feat[GSB_POINTS_THREADS / 32][32 * PT_ROW];
    __shared__ float s_xyz[GSB_POINTS_THREADS / 32][96];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float *const my_feat = &s_feat[warp][lane * PT_ROW];
    float *const my_xyz = &s_xyz[warp][lane * 3];
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long base = (long long)blockIdx.x * blockDim.x + warp * 32; base < p.N; base += stride) {
        const long long id = base + lane;
        if (id < p.N) {
            float4 *gf = reinterpret_cast<float4 *>(my_feat);
            if (PART != 1) {
                const float4 *srow = reinterpret_cast<const float4 *>(p.grad_sum + 12 * (size_t)id);
                const float4 s0 = __ldg(srow), s1 = __ldg(srow + 1), s2 = __ldg(srow + 2);
                my_xyz[0] = s0.x; my_xyz[1] = s0.y; my_xyz[2] = s0.z;
                gf[0] = make_float4(s0.w, s1.x, s1.y, s1.z);
                gf[1] = make_float4(s1.w, s2.x, s2.y, s2.z);
            }
            if (PART != 2) {
            float acc[3][16];
#pragma unroll
            for (int ch = 0; ch < 3; ++ch)
#pragma unroll
                for (int k = 0; k < 16; ++k) acc[ch][k] = 0.0f;
            const float x = p.xyz[3 * (size_t)id], y = p.xyz[3 * (size_t)id + 1], z = p.xyz[3 * (size_t)id + 2];
            const int ob = p.obj_id[id];
#pragma unroll 1
            for (int v = 0; v < p.R; ++v) {
                const float *blk = p.grad_color_views + (size_t)v * p.view_stride;
                const float g[3] = {__ldg(blk + 3 * (size_t)id), __ldg(blk + 3 * (size_t)id + 1), __ldg(blk + 3 * (size_t)id + 2)};
                if (g[0] == 0.0f && g[1] == 0.0f && g[2] == 0.0f) continue;  // outside this view's frustum
                const float *centre = blk + 3 * (size_t)p.N + 3 * ob;
                float sh[16];
                sh_basis(x - __ldg(centre), y - __ldg(centre + 1), z - __ldg(centre + 2), sh);
#pragma unroll
                for (int ch = 0; ch < 3; ++ch)
#pragma unroll
                    for (int k = 0; k < 16; ++k) acc[ch][k] += g[ch] * sh[k] * (k == 0 ? p.c_f : p.h_f);
            }
#pragma unroll
            for (int ch = 0; ch < 3; ++ch)
#pragma unroll
                for (int k4 = 0; k4 < 4; ++k4)
                    gf[2 + 4 * ch + k4] = make_float4(4 * k4 < p.first_cleared ? acc[ch][4 * k4] : 0.0f,
                                                      4 * k4 + 1 < p.first_cleared ? acc[ch][4 * k4 + 1] : 0.0f,
                                                      4 * k4 + 2 < p.first_cleared ? acc[ch][4 * k4 + 2] : 0.0f,
                                                      4 * k4 + 3 < p.first_cleared ? acc[ch][4 * k4 + 3] : 0.0f);
            }
        }
        __syncwarp();
        const long long rows = p.N - base < 32 ? p.N - base : 32;
        float4 *const out_f = reinterpret_cast<float4 *>(p.grad_feat + (size_t)GSB_FEATURE_DIM * base);
#pragma unroll
        for (int it = 0; it < GSB_FEATURE_DIM / 4; ++it) {
            const int f = it * 32 + lane;
            const int row = f / (GSB_FEATURE_DIM / 4), c4 = f - row * (GSB_FEATURE_DIM / 4);
            const bool mine = PART == 0 || (PART == 1 ? c4 >= 2 : c4 < 2);  // float4 0..1 = q s logit, 2..13 = SH
            if (row < rows && mine) out_f[f] = *reinterpret_cast<const float4 *>(&s_feat[warp][row * PT_ROW + 4 * c4]);
        }
        if (PART != 1) {
            float *const out_x = p.grad_xyz + 3 * (size_t)base;
#pragma unroll
            for (int it = 0; it < 3; ++it) {
                const int f = it * 32 + lane;
                if (f < 3 * rows) out_x[f] = s_xyz[warp][f];
            }
        }
        __syncwarp();
    }
}

#ifndef GSB_HOST_EMU
static int first_cleared_of_band(int band) { return band <= 0 ? 1 : band == 1 ? 4 : band == 2 ? 9 : 16; }

static PointsBwdParams make_points_params(const GsbBackwardArgs &a, const Workspace &ws, const long long *skip_flag) {
    PointsBwdParams p;
    p.ctl_num_in_camera = a.ctl_accumulated_num_in_camera;
    p.ctl_num_pixels = a.ctl_accumulated_num_pixels;
    p.ctl_vs_grad = a.ctl_accumulated_view_space_position_gradients;
    p.ctl_vs_grad_avg = a.ctl_accumulated_view_space_position_gradients_avg;
    p.ctl_pos_grad = a.ctl_accumulated_position_gradients;
    p.ctl_pos_grad_norm = a.ctl_accumulated_position_gradients_norm;
    p.skip_flag = skip_flag;
    p.N = a.num_points;
    p.point_offset = ws.point_offset;
    p.records = ws.records;
    p.point_in_camera = ws.point_in_camera;
    p.accum = a.accum;
    p.poses = ws.poses;
    p.xyz = a.pointcloud;
    p.features = a.pointcloud_features;
    p.obj_id = a.point_object_id;
    p.t_pc_cam = a.t_pointcloud_camera;
    p.K = a.camera_intrinsics;
    p.first_cleared = first_cleared_of_band(a.color_max_sh_band);
    p.q_f = a.grad_q_factor;
    p.s_f = a.grad_s_factor;
    p.a_f = a.grad_alpha_factor;
    p.c_f = a.grad_color_factor;
    p.h_f = a.grad_high_order_color_factor;
    p.grad_xyz = a.grad_pointcloud;
    p.grad_feat = a.grad_pointcloud_features;
    p.grad_sum_compact = a.grad_sum_compact;
    p.grad_color_compact = a.grad_color_compact;
    return p;
}

int launch_backward_points(const GsbBackwardArgs &a, const Workspace &ws, cudaStream_t stream, const long long *skip_flag,
                           bool depth_grad) {
    if (a.num_points <= 0) return GSB_OK;
    const PointsBwdParams p = make_points_params(a, ws, skip_flag);
    long long blocks = (a.num_points + GSB_POINTS_THREADS - 1) / GSB_POINTS_THREADS;
    const long long cap = 16LL * num_sms();
    if (blocks > cap) blocks = cap;
    if (blocks <= 0) return GSB_OK;
    const bool compact = (a.flags & GSB_FLAG_COMPACT_GRADS) != 0;
    if (depth_grad) {
        if (compact) backward_points_kernel<true, true><<<(int)blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
        else backward_points_kernel<false, true><<<(int)blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
    } else if (compact) {
        backward_points_kernel<true><<<(int)blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
    } else {
        backward_points_kernel<false><<<(int)blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
    }
    GSB_CUDA_CHECK(cudaGetLastError());
    return GSB_OK;
}

int launch_backward_points_equirect(const GsbBackwardArgs &a, const Workspace &ws, cudaStream_t stream, bool depth_grad) {
    if (a.num_points <= 0) return GSB_OK;
    const PointsBwdParams p = make_points_params(a, ws, nullptr);
    long long blocks = (a.num_points + GSB_POINTS_THREADS - 1) / GSB_POINTS_THREADS;
    const long long cap = 16LL * num_sms();
    if (blocks > cap) blocks = cap;
    if (depth_grad) backward_points_equirect_kernel<true><<<(int)blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
    else backward_points_equirect_kernel<false><<<(int)blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
    GSB_CUDA_CHECK(cudaGetLastError());
    return GSB_OK;
}

int launch_backward_points_lens(const GsbBackwardArgs &a, const Workspace &ws, cudaStream_t stream, bool depth_grad,
                                const LensParams &lens) {
    if (a.num_points <= 0) return GSB_OK;
    PointsBwdLensParams p;
    static_cast<PointsBwdParams &>(p) = make_points_params(a, ws, nullptr);
    p.lens = lens;
    long long blocks = (a.num_points + GSB_POINTS_THREADS - 1) / GSB_POINTS_THREADS;
    const long long cap = 16LL * num_sms();
    if (blocks > cap) blocks = cap;
    if (depth_grad) backward_points_lens_kernel<true><<<(int)blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
    else backward_points_lens_kernel<false><<<(int)blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
    GSB_CUDA_CHECK(cudaGetLastError());
    return GSB_OK;
}

// The LGRAD per-point kernel on a grid that depends on N alone (at most GSB_LENS_GRAD_PARTIAL_BLOCKS CTAs), so the
// summation order of the coefficient gradient is the same on every device, then lens_grad_finish_kernel.  The caller checked
// `lens_grad`.
int launch_backward_points_lens_grad(const GsbBackwardArgs &a, const Workspace &ws, cudaStream_t stream, bool depth_grad,
                                     const LensParams &lens, const GsbLensGradArgs &lens_grad) {
    PointsBwdLensGradParams p;
    static_cast<PointsBwdParams &>(p) = make_points_params(a, ws, nullptr);
    p.lens = lens;
    p.lens_partials = static_cast<float *>(lens_grad.temp);
    long long blocks = a.num_points > 0 ? (a.num_points + GSB_POINTS_THREADS - 1) / GSB_POINTS_THREADS : 0;
    if (blocks > GSB_LENS_GRAD_PARTIAL_BLOCKS) blocks = GSB_LENS_GRAD_PARTIAL_BLOCKS;
    if (blocks > 0) {
        if (depth_grad) backward_points_lens_grad_kernel<true><<<(int)blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
        else backward_points_lens_grad_kernel<false><<<(int)blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
        GSB_CUDA_CHECK(cudaGetLastError());
    }
    lens_grad_finish_kernel<<<1, LENS_GRAD_FINISH_THREADS, 0, stream>>>(p.lens_partials, (int)blocks,
                                                                         lens_grad.grad_coefficients);
    GSB_CUDA_CHECK(cudaGetLastError());
    return GSB_OK;
}

template <bool DEPTH, bool LENS>
static void launch_rs_kernel(bool mgrad, int blocks, cudaStream_t stream, const PointsBwdRsParams &p) {
    if (mgrad) backward_points_rs_kernel<DEPTH, LENS, true><<<blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
    else backward_points_rs_kernel<DEPTH, LENS, false><<<blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
}

// The RS per-point kernel: without rs_grad on the grid of launch_backward_points_lens; with rs_grad (MGRAD) on a grid that
// depends on N alone (at most GSB_RS_GRAD_PARTIAL_BLOCKS CTAs), so the summation order of the motion gradient is the same on
// every device, then rolling_shutter_grad_finish_kernel.  Every per-row output is written by the row's own thread, so it does
// not depend on the grid.  The caller checked the arguments.
int launch_backward_points_rs(const GsbBackwardArgs &a, const Workspace &ws, cudaStream_t stream, bool depth_grad,
                              const LensParams *lens, const RsParams &rs, const GsbRollingShutterGradArgs *rs_grad) {
    PointsBwdRsParams p;
    static_cast<PointsBwdParams &>(p) = make_points_params(a, ws, nullptr);
    p.lens = lens != nullptr ? *lens : LensParams();
    p.rs = rs;
    p.rs_partials = rs_grad != nullptr ? static_cast<float *>(rs_grad->temp) : nullptr;
    long long blocks = a.num_points > 0 ? (a.num_points + GSB_POINTS_THREADS - 1) / GSB_POINTS_THREADS : 0;
    const long long cap = rs_grad != nullptr ? (long long)GSB_RS_GRAD_PARTIAL_BLOCKS : 16LL * num_sms();
    if (blocks > cap) blocks = cap;
    if (blocks > 0) {
        const bool mgrad = rs_grad != nullptr;
        if (lens != nullptr) {
            if (depth_grad) launch_rs_kernel<true, true>(mgrad, (int)blocks, stream, p);
            else launch_rs_kernel<false, true>(mgrad, (int)blocks, stream, p);
        } else {
            if (depth_grad) launch_rs_kernel<true, false>(mgrad, (int)blocks, stream, p);
            else launch_rs_kernel<false, false>(mgrad, (int)blocks, stream, p);
        }
        GSB_CUDA_CHECK(cudaGetLastError());
    }
    if (rs_grad != nullptr) {
        rolling_shutter_grad_finish_kernel<<<1, RS_GRAD_FINISH_THREADS, 0, stream>>>(p.rs_partials, (int)blocks,
                                                                                     rs_grad->grad_motion);
        GSB_CUDA_CHECK(cudaGetLastError());
    }
    return GSB_OK;
}

// mode 0: BLUR, 1: BGRAD, 2: DEFOCUS, 3: DEFOCUS and DGRAD
template <bool DEPTH, bool LENS, bool RS>
static void launch_blur_kernel(int mode, int blocks, cudaStream_t stream, const PointsBwdBlurParams &p) {
    if (mode == 1) backward_points_blur_kernel<DEPTH, LENS, RS, true><<<blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
    else if (mode == 2) backward_points_blur_kernel<DEPTH, LENS, RS, false, true, false><<<blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
    else if (mode == 3) backward_points_blur_kernel<DEPTH, LENS, RS, false, true, true><<<blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
    else backward_points_blur_kernel<DEPTH, LENS, RS, false><<<blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
}

// The BLUR per-point kernel on the grid of launch_backward_points_rs (at most GSB_RS_GRAD_PARTIAL_BLOCKS CTAs with blur_grad
// or defocus_grad), then with either rolling_shutter_grad_finish_kernel.  With defocus_grad the finished row goes to the slot
// after the per-CTA rows in defocus_grad->temp and its first two values (dL/da, dL/drho) to defocus_grad->grad.  The caller
// checked the arguments.
int launch_backward_points_blur(const GsbBackwardArgs &a, const Workspace &ws, cudaStream_t stream, bool depth_grad,
                                const LensParams *lens, const RsParams *rs, const BlurParams &blur,
                                const GsbMotionBlurGradArgs *blur_grad, const DefocusParams *defocus,
                                const GsbDefocusGradArgs *defocus_grad) {
    PointsBwdBlurParams p;
    static_cast<PointsBwdParams &>(p) = make_points_params(a, ws, nullptr);
    p.lens = lens != nullptr ? *lens : LensParams();
    p.rs = rs != nullptr ? *rs : RsParams();
    p.rs_partials = blur_grad != nullptr ? static_cast<float *>(blur_grad->temp)
                    : defocus_grad != nullptr ? static_cast<float *>(defocus_grad->temp) : nullptr;
    p.blur = blur;
    p.defocus = defocus != nullptr ? *defocus : DefocusParams();
    const bool cam_grad = blur_grad != nullptr || defocus_grad != nullptr;
    long long blocks = a.num_points > 0 ? (a.num_points + GSB_POINTS_THREADS - 1) / GSB_POINTS_THREADS : 0;
    const long long cap = cam_grad ? (long long)GSB_RS_GRAD_PARTIAL_BLOCKS : 16LL * num_sms();
    if (blocks > cap) blocks = cap;
    if (blocks > 0) {
        const int mode = defocus != nullptr ? (defocus_grad != nullptr ? 3 : 2) : blur_grad != nullptr ? 1 : 0;
        const bool l = lens != nullptr, r = rs != nullptr;
        const int g = (int)blocks;
        if (depth_grad) {
            if (l) r ? launch_blur_kernel<true, true, true>(mode, g, stream, p) : launch_blur_kernel<true, true, false>(mode, g, stream, p);
            else r ? launch_blur_kernel<true, false, true>(mode, g, stream, p) : launch_blur_kernel<true, false, false>(mode, g, stream, p);
        } else {
            if (l) r ? launch_blur_kernel<false, true, true>(mode, g, stream, p) : launch_blur_kernel<false, true, false>(mode, g, stream, p);
            else r ? launch_blur_kernel<false, false, true>(mode, g, stream, p) : launch_blur_kernel<false, false, false>(mode, g, stream, p);
        }
        GSB_CUDA_CHECK(cudaGetLastError());
    }
    if (cam_grad) {
        float *const row = blur_grad != nullptr ? blur_grad->grad_motion
                                                : p.rs_partials + (size_t)GSB_RS_GRAD_PARTIAL_BLOCKS * RS_GRAD_VALUES;
        rolling_shutter_grad_finish_kernel<<<1, RS_GRAD_FINISH_THREADS, 0, stream>>>(p.rs_partials, (int)blocks, row);
        GSB_CUDA_CHECK(cudaGetLastError());
        if (defocus_grad != nullptr)
            GSB_CUDA_CHECK(cudaMemcpyAsync(defocus_grad->grad, row, 2 * sizeof(float), cudaMemcpyDeviceToDevice, stream));
    }
    return GSB_OK;
}

// The FILTER per-point kernels on the grid of launch_backward_points (lens: NULL for a pinhole; rs: NULL for a global
// shutter); skip_flag as in launch_backward_points.  The caller checked the arguments.
int launch_backward_points_filter(const GsbBackwardArgs &a, const Workspace &ws, cudaStream_t stream, const long long *skip_flag,
                                  bool depth_grad, const LensParams *lens, const RsParams *rs, const float *filter3d) {
    if (a.num_points <= 0) return GSB_OK;
    long long blocks = (a.num_points + GSB_POINTS_THREADS - 1) / GSB_POINTS_THREADS;
    const long long cap = 16LL * num_sms();
    if (blocks > cap) blocks = cap;
    const int g = (int)blocks;
    if (rs != nullptr) {
        PointsBwdRsFilterParams p;
        static_cast<PointsBwdParams &>(p) = make_points_params(a, ws, skip_flag);
        p.lens = lens != nullptr ? *lens : LensParams();
        p.rs = *rs;
        p.rs_partials = nullptr;
        p.filter3d = filter3d;
        if (lens != nullptr) {
            if (depth_grad) backward_points_rs_filter_kernel<true, true><<<g, GSB_POINTS_THREADS, 0, stream>>>(p);
            else backward_points_rs_filter_kernel<false, true><<<g, GSB_POINTS_THREADS, 0, stream>>>(p);
        } else {
            if (depth_grad) backward_points_rs_filter_kernel<true, false><<<g, GSB_POINTS_THREADS, 0, stream>>>(p);
            else backward_points_rs_filter_kernel<false, false><<<g, GSB_POINTS_THREADS, 0, stream>>>(p);
        }
    } else {
        PointsBwdFilterParams p;
        static_cast<PointsBwdParams &>(p) = make_points_params(a, ws, skip_flag);
        p.lens = lens != nullptr ? *lens : LensParams();
        p.filter3d = filter3d;
        if (lens != nullptr) {
            if (depth_grad) backward_points_filter_kernel<true, true><<<g, GSB_POINTS_THREADS, 0, stream>>>(p);
            else backward_points_filter_kernel<false, true><<<g, GSB_POINTS_THREADS, 0, stream>>>(p);
        } else {
            if (depth_grad) backward_points_filter_kernel<true, false><<<g, GSB_POINTS_THREADS, 0, stream>>>(p);
            else backward_points_filter_kernel<false, false><<<g, GSB_POINTS_THREADS, 0, stream>>>(p);
        }
    }
    GSB_CUDA_CHECK(cudaGetLastError());
    return GSB_OK;
}

// The POSE per-point kernel on a grid that depends on N alone (at most GSB_POSE_PARTIAL_BLOCKS CTAs), so the summation
// order of the pose gradient is the same on every device, then pose_finish_kernel.  The caller checked `pose`.
int launch_backward_points_pose(const GsbBackwardArgs &a, const Workspace &ws, cudaStream_t stream, bool depth_grad,
                                const GsbPoseGradArgs &pose) {
    PointsBwdPoseParams p;
    static_cast<PointsBwdParams &>(p) = make_points_params(a, ws, nullptr);
    p.pose_partials = static_cast<float *>(pose.temp);
    p.num_objects = a.num_objects;
    long long blocks = a.num_points > 0 ? (a.num_points + GSB_POINTS_THREADS - 1) / GSB_POINTS_THREADS : 0;
    if (blocks > GSB_POSE_PARTIAL_BLOCKS) blocks = GSB_POSE_PARTIAL_BLOCKS;
    if (blocks > 0) {
        if (depth_grad) backward_points_pose_kernel<true><<<(int)blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
        else backward_points_pose_kernel<false><<<(int)blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
        GSB_CUDA_CHECK(cudaGetLastError());
    }
    pose_finish_kernel<<<a.num_objects, POSE_FINISH_THREADS, 0, stream>>>(
        p.pose_partials, (int)blocks, a.num_objects, pose.q_pointcloud_camera, a.t_pointcloud_camera,
        pose.grad_q_pointcloud_camera, pose.grad_t_pointcloud_camera);
    GSB_CUDA_CHECK(cudaGetLastError());
    return GSB_OK;
}

// The INTR per-point kernel (with the pose sums too when `pose` is set: one pass) on the POSE kernel's grid, then the
// finishing kernels.  The caller checked `pose` and `intr`.
int launch_backward_points_calib(const GsbBackwardArgs &a, const Workspace &ws, cudaStream_t stream, bool depth_grad,
                                 const GsbPoseGradArgs *pose, const GsbIntrinsicsGradArgs &intr) {
    static_assert(GSB_INTRINSICS_PARTIAL_BLOCKS == GSB_POSE_PARTIAL_BLOCKS, "the combined kernel has one grid");
    PointsBwdCalibParams p;
    static_cast<PointsBwdParams &>(p) = make_points_params(a, ws, nullptr);
    p.pose_partials = pose ? static_cast<float *>(pose->temp) : nullptr;
    p.num_objects = pose ? a.num_objects : 0;
    p.intr_partials = static_cast<float *>(intr.temp);
    long long blocks = a.num_points > 0 ? (a.num_points + GSB_POINTS_THREADS - 1) / GSB_POINTS_THREADS : 0;
    if (blocks > GSB_INTRINSICS_PARTIAL_BLOCKS) blocks = GSB_INTRINSICS_PARTIAL_BLOCKS;
    if (blocks > 0) {
        if (pose) {
            if (depth_grad) backward_points_calib_kernel<true, true><<<(int)blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
            else backward_points_calib_kernel<false, true><<<(int)blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
        } else {
            if (depth_grad) backward_points_calib_kernel<true, false><<<(int)blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
            else backward_points_calib_kernel<false, false><<<(int)blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
        }
        GSB_CUDA_CHECK(cudaGetLastError());
    }
    if (pose) {
        pose_finish_kernel<<<a.num_objects, POSE_FINISH_THREADS, 0, stream>>>(
            p.pose_partials, (int)blocks, a.num_objects, pose->q_pointcloud_camera, a.t_pointcloud_camera,
            pose->grad_q_pointcloud_camera, pose->grad_t_pointcloud_camera);
        GSB_CUDA_CHECK(cudaGetLastError());
    }
    intrinsics_finish_kernel<<<1, INTR_FINISH_THREADS, 0, stream>>>(p.intr_partials, (int)blocks,
                                                                     intr.grad_camera_intrinsics);
    GSB_CUDA_CHECK(cudaGetLastError());
    return GSB_OK;
}

template <bool DEPTH>
static void launch_ortho_kernel(bool pose, bool intr, bool filter, int blocks, cudaStream_t stream,
                                const PointsBwdOrthoParams &p) {
    if (filter) backward_points_ortho_kernel<DEPTH, false, false, true><<<blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
    else if (pose && intr) backward_points_ortho_kernel<DEPTH, true, true, false><<<blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
    else if (pose) backward_points_ortho_kernel<DEPTH, true, false, false><<<blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
    else if (intr) backward_points_ortho_kernel<DEPTH, false, true, false><<<blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
    else backward_points_ortho_kernel<DEPTH, false, false, false><<<blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
}

// The ORTHO per-point kernel: without camera gradients on the grid of launch_backward_points; with pose or intrinsics on the
// POSE kernel's grid (it depends on N alone), then the finishing kernels, as launch_backward_points_calib.  filter3d never comes
// with pose or intr.  The caller checked the arguments.
int launch_backward_points_ortho(const GsbBackwardArgs &a, const Workspace &ws, cudaStream_t stream, bool depth_grad,
                                 const GsbPoseGradArgs *pose, const GsbIntrinsicsGradArgs *intr, const float *filter3d) {
    PointsBwdOrthoParams p;
    static_cast<PointsBwdParams &>(p) = make_points_params(a, ws, nullptr);
    p.pose_partials = pose ? static_cast<float *>(pose->temp) : nullptr;
    p.num_objects = pose ? a.num_objects : 0;
    p.intr_partials = intr ? static_cast<float *>(intr->temp) : nullptr;
    p.filter3d = filter3d;
    const bool cam_grad = pose != nullptr || intr != nullptr;
    long long blocks = a.num_points > 0 ? (a.num_points + GSB_POINTS_THREADS - 1) / GSB_POINTS_THREADS : 0;
    const long long cap = cam_grad ? (long long)GSB_POSE_PARTIAL_BLOCKS : 16LL * num_sms();
    if (blocks > cap) blocks = cap;
    if (blocks > 0) {
        const bool f = filter3d != nullptr;
        if (depth_grad) launch_ortho_kernel<true>(pose != nullptr, intr != nullptr, f, (int)blocks, stream, p);
        else launch_ortho_kernel<false>(pose != nullptr, intr != nullptr, f, (int)blocks, stream, p);
        GSB_CUDA_CHECK(cudaGetLastError());
    }
    if (pose) {
        pose_finish_kernel<<<a.num_objects, POSE_FINISH_THREADS, 0, stream>>>(
            p.pose_partials, (int)blocks, a.num_objects, pose->q_pointcloud_camera, a.t_pointcloud_camera,
            pose->grad_q_pointcloud_camera, pose->grad_t_pointcloud_camera);
        GSB_CUDA_CHECK(cudaGetLastError());
    }
    if (intr) {
        intrinsics_finish_kernel<<<1, INTR_FINISH_THREADS, 0, stream>>>(p.intr_partials, (int)blocks,
                                                                         intr->grad_camera_intrinsics);
        GSB_CUDA_CHECK(cudaGetLastError());
    }
    return GSB_OK;
}

template <bool DEPTH>
static void launch_lens_calib_kernel(bool pose, bool intr, bool lgrad, int blocks, cudaStream_t stream,
                                     const PointsBwdLensCalibParams &p) {
    if (pose && intr && lgrad) backward_points_lens_calib_kernel<DEPTH, true, true, true><<<blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
    else if (pose && intr) backward_points_lens_calib_kernel<DEPTH, true, true, false><<<blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
    else if (pose && lgrad) backward_points_lens_calib_kernel<DEPTH, true, false, true><<<blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
    else if (pose) backward_points_lens_calib_kernel<DEPTH, true, false, false><<<blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
    else if (lgrad) backward_points_lens_calib_kernel<DEPTH, false, true, true><<<blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
    else backward_points_lens_calib_kernel<DEPTH, false, true, false><<<blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
}

// The LENS per-point kernel with pose and / or intrinsics sums (and the coefficient sums with lens_grad) on the POSE kernel's
// grid (it depends on N alone), then the finishing kernels of launch_backward_points_calib and
// launch_backward_points_lens_grad.  Every per-row output is written by the row's own thread, as in the LENS kernel.  The
// caller checked the arguments (pose or intr is set).
int launch_backward_points_lens_calib(const GsbBackwardArgs &a, const Workspace &ws, cudaStream_t stream, bool depth_grad,
                                      const LensParams &lens, const GsbLensGradArgs *lens_grad, const GsbPoseGradArgs *pose,
                                      const GsbIntrinsicsGradArgs *intr) {
    static_assert(GSB_INTRINSICS_PARTIAL_BLOCKS == GSB_POSE_PARTIAL_BLOCKS &&
                  GSB_LENS_GRAD_PARTIAL_BLOCKS == GSB_POSE_PARTIAL_BLOCKS, "the combined kernel has one grid");
    PointsBwdLensCalibParams p;
    static_cast<PointsBwdParams &>(p) = make_points_params(a, ws, nullptr);
    p.pose_partials = pose ? static_cast<float *>(pose->temp) : nullptr;
    p.num_objects = pose ? a.num_objects : 0;
    p.intr_partials = intr ? static_cast<float *>(intr->temp) : nullptr;
    p.lens = lens;
    p.lens_partials = lens_grad ? static_cast<float *>(lens_grad->temp) : nullptr;
    long long blocks = a.num_points > 0 ? (a.num_points + GSB_POINTS_THREADS - 1) / GSB_POINTS_THREADS : 0;
    if (blocks > GSB_POSE_PARTIAL_BLOCKS) blocks = GSB_POSE_PARTIAL_BLOCKS;
    if (blocks > 0) {
        const bool ps = pose != nullptr, in = intr != nullptr, lg = lens_grad != nullptr;
        if (depth_grad) launch_lens_calib_kernel<true>(ps, in, lg, (int)blocks, stream, p);
        else launch_lens_calib_kernel<false>(ps, in, lg, (int)blocks, stream, p);
        GSB_CUDA_CHECK(cudaGetLastError());
    }
    if (pose) {
        pose_finish_kernel<<<a.num_objects, POSE_FINISH_THREADS, 0, stream>>>(
            p.pose_partials, (int)blocks, a.num_objects, pose->q_pointcloud_camera, a.t_pointcloud_camera,
            pose->grad_q_pointcloud_camera, pose->grad_t_pointcloud_camera);
        GSB_CUDA_CHECK(cudaGetLastError());
    }
    if (intr) {
        intrinsics_finish_kernel<<<1, INTR_FINISH_THREADS, 0, stream>>>(p.intr_partials, (int)blocks,
                                                                         intr->grad_camera_intrinsics);
        GSB_CUDA_CHECK(cudaGetLastError());
    }
    if (lens_grad) {
        lens_grad_finish_kernel<<<1, LENS_GRAD_FINISH_THREADS, 0, stream>>>(p.lens_partials, (int)blocks,
                                                                             lens_grad->grad_coefficients);
        GSB_CUDA_CHECK(cudaGetLastError());
    }
    return GSB_OK;
}

int launch_expand_view_gradients(const GsbExpandArgs &a, cudaStream_t stream) {
    if (a.num_points <= 0) return GSB_OK;
    ExpandParams p;
    p.N = a.num_points;
    p.R = a.num_views;
    p.grad_sum = a.grad_sum;
    p.grad_color_views = a.grad_color_views;
    p.view_stride = a.view_stride;
    p.xyz = a.pointcloud;
    p.obj_id = a.point_object_id;
    p.first_cleared = first_cleared_of_band(a.color_max_sh_band);
    p.c_f = a.grad_color_factor;
    p.h_f = a.grad_high_order_color_factor;
    p.grad_xyz = a.grad_pointcloud;
    p.grad_feat = a.grad_pointcloud_features;
    long long blocks = (a.num_points + GSB_POINTS_THREADS - 1) / GSB_POINTS_THREADS;
    const long long cap = 16LL * num_sms();
    if (blocks > cap) blocks = cap;
    if (a.part == 1) expand_view_gradients_kernel<1><<<(int)blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
    else if (a.part == 2) expand_view_gradients_kernel<2><<<(int)blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
    else expand_view_gradients_kernel<0><<<(int)blocks, GSB_POINTS_THREADS, 0, stream>>>(p);
    GSB_CUDA_CHECK(cudaGetLastError());
    return GSB_OK;
}
#endif  // GSB_HOST_EMU

}  // namespace gsb
