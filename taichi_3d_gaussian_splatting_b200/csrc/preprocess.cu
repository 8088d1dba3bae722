// preprocess.cu -- per-Gaussian stage, ONE pass over the N rows of the scene:
//   frustum filter (GPCR:31-78) + order-preserving compaction (GPCR:861-864)
//   + projection / EWA covariance / conic / opacity / SH colour / radius (GPCR:239-315)
//   + tile-rect count (GPCR:81-128) + exclusive scan of the counts (GPCR:913-922)
//   + (tile, depth) key emission (GPCR:131-172)
// fused behind a single-pass decoupled look-back scan of the pair (in-frustum flag, tile count), so a
// point's in-camera offset and its key range are known inside the same kernel and nothing is re-read.
//
// This translation unit is compiled with -fmad=false: every float op is a plain IEEE op in the same
// order as the CPU oracle, and exp() is evaluated in double and rounded once, so all discrete per-point
// decisions (frustum test, tile bbox, depth key) are bit-reproducible.  On paper the stage is HBM-bound (~240 B read,
// ~70 B + 8..12 B/key written per in-frustum point); in practice it is bound by instruction issue and latency (unfused
// IEEE arithmetic, seven exp() in double per point).  Staging each warp's 32 contiguous feature rows (7 KB) with one TMA
// bulk copy was rejected: the extra 28 KB of shared memory per CTA cut the occupancy from 8 to 5 CTAs per SM and the bulk
// copy put the whole row fetch in front of the scan's aggregate publish.
#include "common.cuh"

namespace gsb {

// ------------------------------------------------------------------ small device math (IEEE order)
template <int AR, int AC, int BC>
__device__ __forceinline__ void matmul(const float *a, const float *b, float *out) {
#pragma unroll
    for (int i = 0; i < AR; ++i)
#pragma unroll
        for (int j = 0; j < BC; ++j) {
            float s = a[i * AC] * b[j];
#pragma unroll
            for (int k = 1; k < AC; ++k) s = s + a[i * AC + k] * b[k * BC + j];
            out[i * BC + j] = s;
        }
}

// GP3D:30-48 (xyzw, not re-normalised)
__device__ __forceinline__ void rotation_from_quaternion(float x, float y, float z, float w, float *R) {
    float xx = x * x, yy = y * y, zz = z * z;
    float xy = x * y, xz = x * z, yz = y * z;
    float wx = w * x, wy = w * y, wz = w * z;
    R[0] = 1 - 2 * (yy + zz); R[1] = 2 * (xy - wz);     R[2] = 2 * (xz + wy);
    R[3] = 2 * (xy + wz);     R[4] = 1 - 2 * (xx + zz); R[5] = 2 * (yz - wx);
    R[6] = 2 * (xz - wy);     R[7] = 2 * (yz + wx);     R[8] = 1 - 2 * (xx + yy);
}

__device__ __forceinline__ float exp_cr(float x) { return (float)exp((double)x); }
__device__ __forceinline__ float sigmoid_cr(float x) { return 1.0f / (1.0f + exp_cr(-x)); }

// quaternion product, UT:396-411
__device__ __forceinline__ void quat_mul(const float *a, const float *b, float *o) {
    float x0 = a[0], y0 = a[1], z0 = a[2], w0 = a[3];
    float x1 = b[0], y1 = b[1], z1 = b[2], w1 = b[3];
    o[0] = w0 * x1 + x0 * w1 + y0 * z1 - z0 * y1;
    o[1] = w0 * y1 - x0 * z1 + y0 * w1 + z0 * x1;
    o[2] = w0 * z1 + x0 * y1 - y0 * x1 + z0 * w1;
    o[3] = w0 * w1 - x0 * x1 - y0 * y1 - z0 * z1;
}

// ------------------------------------------------------------------ pose kernel
// inverse_SE3_qt_torch (UT:426-432, called at GPCR:845) + transform_matrix_from_quaternion_and_translation
// (GP3D:51-62) + camera centre of taichi_inverse_SE3 (UT:495-510), once per object instead of per point.
// It is the frame's first kernel, so it also zeroes the two 16-byte-aligned ranges [clear0, clear0 + clear0_vec) and
// [clear1, clear1 + clear1_vec) of per-frame state (counters, tickets, the compaction scan's look-back state, the digit
// histograms, the tile ranges) that the later kernels count into or spin on, so the forward needs no driver memset.  The
// sort's look-back state is cleared by the histogram kernel, which knows the frame's key count.
__global__ void pose_kernel(const float *__restrict__ q_pc, const float *__restrict__ t_pc, int n_obj,
                            PoseBlock *__restrict__ poses, uint4 *__restrict__ clear0 = nullptr, int clear0_vec = 0,
                            uint4 *__restrict__ clear1 = nullptr, int clear1_vec = 0) {
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    const int stride = gridDim.x * blockDim.x;
    for (int k = o; k < clear0_vec; k += stride) clear0[k] = make_uint4(0u, 0u, 0u, 0u);
    for (int k = o; k < clear1_vec; k += stride) clear1[k] = make_uint4(0u, 0u, 0u, 0u);
    if (o >= n_obj) return;
    float qi[4] = {-q_pc[4 * o], -q_pc[4 * o + 1], -q_pc[4 * o + 2], q_pc[4 * o + 3]};
    float t[3] = {t_pc[3 * o], t_pc[3 * o + 1], t_pc[3 * o + 2]};
    float n = sqrtf(((qi[0] * qi[0] + qi[1] * qi[1]) + qi[2] * qi[2]) + qi[3] * qi[3]);
    float qn[4] = {qi[0] / n, qi[1] / n, qi[2] / n, qi[3] / n};
    float v[4] = {t[0], t[1], t[2], 0.0f};
    float qc[4] = {-qn[0], -qn[1], -qn[2], qn[3]};
    float tmp[4], rot[4];
    quat_mul(qn, v, tmp);
    quat_mul(tmp, qc, rot);
    float ti[3] = {-rot[0], -rot[1], -rot[2]};
    float R[9];
    rotation_from_quaternion(qi[0], qi[1], qi[2], qi[3], R);
    PoseBlock pb;
    pb.T[0] = R[0]; pb.T[1] = R[1]; pb.T[2] = R[2];  pb.T[3] = ti[0];
    pb.T[4] = R[3]; pb.T[5] = R[4]; pb.T[6] = R[5];  pb.T[7] = ti[1];
    pb.T[8] = R[6]; pb.T[9] = R[7]; pb.T[10] = R[8]; pb.T[11] = ti[2];
    float nRT[9] = {-R[0], -R[3], -R[6], -R[1], -R[4], -R[7], -R[2], -R[5], -R[8]};
    matmul<3, 3, 1>(nRT, ti, pb.centre);
#pragma unroll
    for (int k = 0; k < 5; ++k) pb.pad[k] = 0.0f;
    poses[o] = pb;
}

// ------------------------------------------------------------------ look-back scan state
// 64-bit word: [63:62] status, [61:36] point count (26 b), [35:0] tile-pair count (36 b).
constexpr unsigned long long ST_AGGREGATE = 1ull << 62;
constexpr unsigned long long ST_INCLUSIVE = 2ull << 62;
constexpr unsigned long long ST_VALUE_MASK = (1ull << 62) - 1;
constexpr int CNT_SHIFT = 36;

__device__ __forceinline__ unsigned long long ld_state(const unsigned long long *p) {
    return *reinterpret_cast<const volatile unsigned long long *>(p);
}
__device__ __forceinline__ void st_state(unsigned long long *p, unsigned long long v) {
    *reinterpret_cast<volatile unsigned long long *>(p) = v;
}

__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long v) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    return v;
}

struct PreParams {
    long long N;
    const float *xyz;
    float *features;
    const signed char *invalid;
    const int *obj_id;
    const PoseBlock *poses;
    const float *K;
    int W, H;
    float near_plane, far_plane, depth_scale;
    int depth_bits;
    int skip_q_normalise;
    int filter_tiles;
    long long key_capacity;
    long long key_store_limit;  // padded capacity of the key buffers: every slot the sort may read gets a valid key
    int num_blocks;
    // outputs
    long long *counters;
    unsigned int *tickets;
    unsigned long long *scan_state;
    int *point_id;
    int *point_offset;
    int *num_tiles;
    float4 *records;
    float *point_in_camera;
    void *keys;
    int *vals;
};

// GPCR:81-103
__device__ __forceinline__ void bounding_box(float u, float v, float radii, int W, int H, int &a, int &b,
                                             int &c, int &d) {
    radii = fmaxf(radii, 1.0f);
    float min_u = fmaxf(0.0f, u - radii), max_u = u + radii;
    float min_v = fmaxf(0.0f, v - radii), max_v = v + radii;
    int tw = W / GSB_TILE_WIDTH, th = H / GSB_TILE_HEIGHT;
    a = min((int)floorf(min_u / (float)GSB_TILE_WIDTH), tw);
    b = min(max((int)floorf(max_u / (float)GSB_TILE_WIDTH) + 1, a + 1), tw);
    c = min((int)floorf(min_v / (float)GSB_TILE_HEIGHT), th);
    d = min(max((int)floorf(max_v / (float)GSB_TILE_HEIGHT) + 1, c + 1), th);
}

// The tile columns [a, b) of an equirectangular footprint (u in [0, W)): not clamped to the image, and a footprint wider than
// the panorama is cut to the W/16 columns whose centres lie within W/2 of u, so that every column of the window is the copy
// the blend kernels stage the splat at (equirect_wrap_u).  NaN or inf radii take the whole row.
__device__ __forceinline__ void equirect_columns(float u, float radii, int W, int &a, int &b) {
    radii = fmaxf(radii, 1.0f);
    const int tw = W / GSB_TILE_WIDTH;
    const float fa = floorf((u - radii) / (float)GSB_TILE_WIDTH), fb = floorf((u + radii) / (float)GSB_TILE_WIDTH) + 1.0f;
    if (fb - fa <= (float)tw) {
        a = (int)fa;
        b = (int)fb;
    } else {
        a = (int)ceilf((u - 0.5f * (float)W - 0.5f * (float)GSB_TILE_WIDTH) / (float)GSB_TILE_WIDTH);
        b = a + tw;
    }
}

#ifndef GSB_PRE_MIN_BLOCKS
#define GSB_PRE_MIN_BLOCKS 5
#endif
// Per-warp staging area of the cooperative reach filter / key emission (32 splats of the warp).
struct WarpStage {
    float u[32], v[32], a[32], b2[32], c[32], nb_ic[32], nb_ia[32], t2[32];
    int min_tu[32], min_tv[32], ntv[32];
    unsigned int mask_lo[32], mask_hi[32];  // reachable tiles among the first 64 of the splat's square
    int pref[33];                           // warp prefix of per-splat pair / key counts
    int nk64[32], depth_key[32], off[32];
    long long key_base[32];
};

// position of the j-th (0-based) set bit of m; j < popc(m).  Five popc steps instead of the library's bit loop.
__device__ __forceinline__ int select_bit32(unsigned int m, int j) {
    int pos = 0;
#pragma unroll
    for (int w = 16; w >= 1; w >>= 1) {
        const int c = __popc(m & ((1u << w) - 1u));
        const bool up = j >= c;
        j -= up ? c : 0;
        pos += up ? w : 0;
        m = up ? (m >> w) : m;
    }
    return pos;
}

// pixel centres of tile (tu, tv) relative to the splat centre
__device__ __forceinline__ bool tile_reachable(const SplatReach &r, float u, float v, int tu, int tv) {
    const float X0 = (float)(tu * GSB_TILE_WIDTH) + 0.5f - u;
    const float Y0 = (float)(tv * GSB_TILE_HEIGHT) + 0.5f - v;
    return rect_reachable(r, X0, X0 + (float)(GSB_TILE_WIDTH - 1), Y0, Y0 + (float)(GSB_TILE_HEIGHT - 1));
}

// The body of the per-point kernel.  LENS = GSB_LENS_PINHOLE is the default kernel; GSB_LENS_OPENCV / GSB_LENS_FISHEYE
// (gsb200_forward_lens) project through lens_distort (common.cuh): the position is (K00 xd + K01 yd + K02, K10 xd + K11 yd +
// K12), J = diag(fx, fy) D P, and a point with r^2 > lens.r2_max is outside the frustum.  Everything downstream of (u, v) and
// J -- the record layout, the keys, the scan -- is the same for every model.
// ROLLING = true (gsb200_forward_rolling_shutter): the point is moved to its row time first (definition in include/gsb200.h).  The
// GSB_RS_ITERATIONS fixed-point steps project pc(tau_k) through the same lens arithmetic as the position below, the point is
// rendered at pc(tau_3), Sigma' uses W_eff = Rd(tau_3) W, and tau_3 (0 outside the frustum) goes to rs.row_time[i].  The SH
// view direction keeps the mid-readout camera centre.
// FILTER = true (gsb200_forward_filter3d): the row's 3D smoothing filter sigma = fmaxf(filter3d[i], 0) (definition in
// include/gsb200.h) widens the scales to s^_j = sqrt(exp(s_j)^2 + sigma^2) before Sigma is formed, and the compensation
// c = sqrt(prod_j exp(s_j)^2 / s^_j^2) is folded into the record's rescale slot (r1.y = rescale c; r1.z keeps the raw
// opacity), so the blend kernels read rescale * o * c unchanged.  sigma = 0 leaves the row untouched.
// BLUR = true (gsb200_forward_motion_blur): the splat is widened by the exposure motion (definition in include/gsb200.h).
// d = Jp (v + w x pc) with the full position Jacobian Jp at the rendered pc, B = d d^T / 12; the conic is (Sigma_d + B)^-1,
// the rescale slot holds rescale c_b with c_b = sqrt(det Sigma_d / det(Sigma_d + B)), and the radius comes from Sigma' + B.
// A view with m = 0 takes the un-blurred arithmetic.  Not with FILTER.
// DEFOCUS = true (with BLUR; gsb200_forward_defocus): B also carries the thin lens' B_d = beta M M^T, beta = a^2 (rho - 1/z)^2
// / 16 at the rendered z, M = K[:2,:2] (K[:2,:2] D with a lens): B = B_m + B_d, and the conic, c_b, radius and reach follow
// from Sigma_d + B as above.  A view with a = 0 takes the arithmetic without defocus.
// LENS = LENS_EQUIRECT (gsb200_forward_equirect): the equirectangular panorama (definition in include/gsb200.h).  (u, v), the
// in-view test and J come from equirect_project / equirect_jacobian (common.cuh), the depth is the ray distance r (record,
// sort key, CNT_MAX_DEPTH_KEY), the footprint's columns from equirect_columns, and the key's tile column is taken modulo
// W/16.  Not with ROLLING, FILTER or BLUR.
// LENS = LENS_ORTHO (gsb200_forward_ortho): the orthographic view (definition in include/gsb200.h).  (u, v) = K[:2] (x, y, 1)
// without a divide, J = K[:2,:2] [I 0], the in-view test and the depth z are the pinhole's, and the SH view direction is the
// camera's forward axis, row 2 of W, for every point.  With or without FILTER; not with ROLLING or BLUR.
template <typename KeyT, int LENS, bool ROLLING = false, bool FILTER = false, bool BLUR = false, bool DEFOCUS = false>
__device__ __forceinline__ void preprocess_body(const PreParams p, const LensParams lens, const RsParams rs = RsParams(),
                                                const float *filter3d = nullptr, const BlurParams blur = BlurParams(),
                                                const DefocusParams defocus = DefocusParams()) {
    static_assert(!(BLUR && FILTER), "the motion blur is not implemented with the 3D filter");
    static_assert(!DEFOCUS || BLUR, "the defocus runs on the motion-blur path");
    constexpr bool EQUIRECT = LENS == LENS_EQUIRECT;
    static_assert(!EQUIRECT || (!ROLLING && !FILTER && !BLUR), "the panorama is implemented without the camera extensions");
    constexpr bool ORTHO = LENS == LENS_ORTHO;
    static_assert(!ORTHO || (!ROLLING && !BLUR), "the orthographic view is implemented without the camera motions");
    __shared__ unsigned int s_ticket;
    __shared__ unsigned long long s_warp_sums[SCAN_BLOCK_THREADS / 32];
    __shared__ unsigned long long s_block_exclusive;
    __shared__ WarpStage s_stage[SCAN_BLOCK_THREADS / 32];

    const int tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_ticket = atomicAdd(&p.tickets[TICKET_SCAN], 1u);
    __syncthreads();
    const int blk = (int)s_ticket;
    const long long i = (long long)blk * SCAN_BLOCK_THREADS + tid;

    bool in = false;
    int ntiles = 0, nkeys = 0, min_tu = 0, max_tu = 0, min_tv = 0, max_tv = 0;
    SplatReach reach;
    reach.a = reach.b2 = reach.c = reach.nb_ic = reach.nb_ia = reach.t2 = 0.0f;
    reach.mode = 2;
    float4 r0 = make_float4(0, 0, 0, 0), r1 = r0, r2 = r0;
    float pc[3] = {0, 0, 0};
    float dir0 = 0.0f, dir1 = 0.0f, dir2 = 0.0f;  // unit view direction (GPCR:302), consumed by the SH stage
    float tau = 0.0f;                             // ROLLING: the row time
    float depth = 0.0f, eq_rho = 0.0f;            // EQUIRECT: the ray distance r and rho = |(x, z)|

    // Every global load of a point that depends on nothing but its index is issued HERE, in one go: the invalid mask, the
    // object id, the position and the first 32 bytes of the feature row (q | s, logit).  The kernel is bound by the latency
    // of a CTA's dependency chain (DESIGN section 3): mask -> object id -> pose -> position -> frustum test -> feature row
    // were four dependent round trips, now they are one plus the (L1-resident) pose.  Rows outside the frustum or unused
    // fetch 32 bytes they do not need (they are allocated:
    // (N,56)); the arithmetic is untouched.
    signed char h_inv = 1;
    int h_ob = 0;
    float h_x = 0.0f, h_y = 0.0f, h_z = 0.0f;
    float4 h_q = make_float4(0, 0, 0, 0), h_sl = h_q;
    float h_sigma = 0.0f;  // FILTER
    if (i < p.N) {
        h_inv = p.invalid[i];
        h_ob = p.obj_id[i];
        h_x = __ldg(&p.xyz[3 * i]);
        h_y = __ldg(&p.xyz[3 * i + 1]);
        h_z = __ldg(&p.xyz[3 * i + 2]);
        const float4 *hrow = reinterpret_cast<const float4 *>(p.features + (size_t)GSB_FEATURE_DIM * i);
        h_q = hrow[0];           // plain load: this thread rewrites the row's q below
        h_sl = __ldg(hrow + 1);  // s0 s1 s2 logit
        if (FILTER) h_sigma = __ldg(&filter3d[i]);
    }
    if (i < p.N && h_inv != 1) {
        const PoseBlock *pb = p.poses + h_ob;
        float T[12];
#pragma unroll
        for (int k = 0; k < 12; ++k) T[k] = __ldg(&pb->T[k]);
        float Kc[9];
#pragma unroll
        for (int k = 0; k < 9; ++k) Kc[k] = __ldg(&p.K[k]);
        const float x = h_x, y = h_y, z = h_z;
        // GP3D:14-27: T @ (x,y,z,1), then uv = (K @ pc) / pc.z
        pc[0] = ((T[0] * x + T[1] * y) + T[2] * z) + T[3] * 1.0f;
        pc[1] = ((T[4] * x + T[5] * y) + T[6] * z) + T[7] * 1.0f;
        pc[2] = ((T[8] * x + T[9] * y) + T[10] * z) + T[11] * 1.0f;
        float Rd[9];  // ROLLING: Rd(tau_3)
        if (ROLLING) {
            const float pc0[3] = {pc[0], pc[1], pc[2]};
#pragma unroll 1
            for (int it = 0; it < GSB_RS_ITERATIONS; ++it) {
                rolling_shutter_rotation(tau, rs.motion + 3, Rd);
                float pt[3];
                rolling_shutter_point(Rd, tau, rs.motion, pc0, pt);
                float vp;  // the row coordinate of pc(tau), as v below
                if (LENS == GSB_LENS_PINHOLE) {
                    vp = ((Kc[3] * pt[0] + Kc[4] * pt[1]) + Kc[5] * pt[2]) / pt[2];
                } else {
                    float ox, oy, Dt[4];
                    lens_distort<LENS>(lens.k, pt[0] / pt[2], pt[1] / pt[2], ox, oy, Dt);
                    vp = ((Kc[3] * (pt[0] + pt[2] * ox) + Kc[4] * (pt[1] + pt[2] * oy)) + Kc[5] * pt[2]) / pt[2];
                }
                tau = fminf(fmaxf(vp / (float)p.H - 0.5f, -0.5f), 0.5f);  // fmaxf(NaN, -1/2) = -1/2
            }
            rolling_shutter_rotation(tau, rs.motion + 3, Rd);
            rolling_shutter_point(Rd, tau, rs.motion, pc0, pc);
        }
        float u, v;
        float D[4] = {1.0f, 0.0f, 0.0f, 1.0f};  // d(xd, yd)/d(xn, yn)
        bool lens_ok = true;
        if (EQUIRECT) {
            in = equirect_project(Kc, p.W, p.near_plane, p.far_plane, pc, u, v, eq_rho, depth) &&
                 v >= (float)(-GSB_TILE_HEIGHT * GSB_BOUNDARY_TILES) &&
                 v < (float)(p.H + GSB_TILE_HEIGHT * GSB_BOUNDARY_TILES);
        } else if (ORTHO) {  // K[:2] (x, y, 1): no divide, K's last row unread
            u = (Kc[0] * pc[0] + Kc[1] * pc[1]) + Kc[2];
            v = (Kc[3] * pc[0] + Kc[4] * pc[1]) + Kc[5];
        } else if (LENS == GSB_LENS_PINHOLE) {
            float uv1[3];
            matmul<3, 3, 1>(Kc, pc, uv1);
            u = uv1[0] / pc[2];
            v = uv1[1] / pc[2];
        } else {
            const float xn = pc[0] / pc[2], yn = pc[1] / pc[2];
            lens_ok = xn * xn + yn * yn <= lens.r2_max;  // NaN (z = 0) fails as well
            float ox, oy;
            lens_distort<LENS>(lens.k, xn, yn, ox, oy, D);
            // u = K00 xd + K01 yd + K02 as (K z (xd, yd, 1))[0] / z, the pinhole's arithmetic on the displaced point
            const float pd[3] = {pc[0] + pc[2] * ox, pc[1] + pc[2] * oy, pc[2]};
            float uv1[3];
            matmul<3, 3, 1>(Kc, pd, uv1);
            u = uv1[0] / pc[2];
            v = uv1[1] / pc[2];
        }
        if (!EQUIRECT) {
            depth = pc[2];
            in = lens_ok && pc[2] > p.near_plane && pc[2] < p.far_plane &&
                 u >= (float)(-GSB_TILE_WIDTH * GSB_BOUNDARY_TILES) &&
                 u < (float)(p.W + GSB_TILE_WIDTH * GSB_BOUNDARY_TILES) &&
                 v >= (float)(-GSB_TILE_HEIGHT * GSB_BOUNDARY_TILES) &&
                 v < (float)(p.H + GSB_TILE_HEIGHT * GSB_BOUNDARY_TILES);
        }
        if (in) {
            float4 *frow = reinterpret_cast<float4 *>(p.features + (size_t)GSB_FEATURE_DIM * i);
            float4 qv = h_q;
            const float4 sl = h_sl;
            const float f[4] = {sl.x, sl.y, sl.z, sl.w};
            // GPCR:196-205: q <- q / |q| (invlen * q), written back in place
            if (!p.skip_q_normalise) {
                float qn = sqrtf(((qv.x * qv.x + qv.y * qv.y) + qv.z * qv.z) + qv.w * qv.w);
                float inv = 1.0f / qn;
                qv.x = inv * qv.x; qv.y = inv * qv.y; qv.z = inv * qv.z; qv.w = inv * qv.w;
                frow[0] = qv;
            }
            // GP3D:161-191: Sigma' = J W R S S^T R^T W^T J^T
            float J[6];
            const float fx = Kc[0], fy = Kc[4];
            J[0] = fx / pc[2]; J[1] = 0.0f; J[2] = -(fx * pc[0]) / (pc[2] * pc[2]);
            J[3] = 0.0f; J[4] = fy / pc[2]; J[5] = -(fy * pc[1]) / (pc[2] * pc[2]);
            if (LENS != GSB_LENS_PINHOLE && !ORTHO) {  // J = diag(fx, fy) D P, P = [1/z 0 -x/z^2; 0 1/z -y/z^2]
                J[0] = (fx * D[0]) / pc[2]; J[1] = (fx * D[1]) / pc[2];
                J[2] = -(fx * (D[0] * pc[0] + D[1] * pc[1])) / (pc[2] * pc[2]);
                J[3] = (fy * D[2]) / pc[2]; J[4] = (fy * D[3]) / pc[2];
                J[5] = -(fy * (D[2] * pc[0] + D[3] * pc[1])) / (pc[2] * pc[2]);
            }
            if (EQUIRECT) equirect_jacobian(fx, fy, pc, eq_rho, depth, J);
            if (ORTHO) {  // J = K[:2,:2] [I 0]
                J[0] = Kc[0]; J[1] = Kc[1]; J[2] = 0.0f;
                J[3] = Kc[3]; J[4] = Kc[4]; J[5] = 0.0f;
            }
            float R[9], S[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, RS[9], RSS[9], RT[9], Sigma[9];
            rotation_from_quaternion(qv.x, qv.y, qv.z, qv.w, R);
            S[0] = exp_cr(f[0]); S[4] = exp_cr(f[1]); S[8] = exp_cr(f[2]);
            float filter_c = 1.0f;  // FILTER: the opacity compensation c
            if (FILTER) {
                const float sg = fmaxf(h_sigma, 0.0f);  // NaN -> 0
                const float s2 = sg * sg;
                if (s2 > 0.0f) {
                    float ratio = 1.0f;
#pragma unroll
                    for (int j = 0; j < 3; ++j) {
                        const float e = S[4 * j] * S[4 * j], eh = e + s2;
                        ratio = ratio * (e / eh);  // a product of ratios in (0, 1]: no overflow
                        S[4 * j] = sqrtf(eh);
                    }
                    filter_c = sqrtf(ratio);
                }
            }
            matmul<3, 3, 3>(R, S, RS);
            matmul<3, 3, 3>(RS, S, RSS);  // S^T == S (diagonal)
#pragma unroll
            for (int a = 0; a < 3; ++a)
#pragma unroll
                for (int b = 0; b < 3; ++b) RT[b * 3 + a] = R[a * 3 + b];
            matmul<3, 3, 3>(RSS, RT, Sigma);
            float Wm[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
            if (ROLLING) {  // W_eff = Rd W
                float We[9];
                matmul<3, 3, 3>(Rd, Wm, We);
#pragma unroll
                for (int k = 0; k < 9; ++k) Wm[k] = We[k];
            }
            float WT[9], JW[6], JWS[6], JWSW[6], JT[6], cov[4];
#pragma unroll
            for (int a = 0; a < 3; ++a)
#pragma unroll
                for (int b = 0; b < 3; ++b) WT[b * 3 + a] = Wm[a * 3 + b];
            matmul<2, 3, 3>(J, Wm, JW);
            matmul<2, 3, 3>(JW, Sigma, JWS);
            matmul<2, 3, 3>(JWS, WT, JWSW);
            JT[0] = J[0]; JT[1] = J[3]; JT[2] = J[1]; JT[3] = J[4]; JT[4] = J[2]; JT[5] = J[5];
            matmul<2, 3, 2>(JWSW, JT, cov);
            // UT:257-272 conic + rescale (+0.3 low-pass)
            float c00 = cov[0], c01 = cov[1], c10 = cov[2], c11 = cov[3];
            const float det_pre = c00 * c11 - c01 * c10;
            c00 += 0.3f;
            c11 += 0.3f;
            float det = c00 * c11 - c01 * c10;
            const float rescale = sqrtf(fmaxf(0.0f, det_pre / det));
            float blur_c = 1.0f;  // BLUR: the compensation c_b
            const bool moving = BLUR && motion_blur_on(blur.motion);
            const bool defocused = DEFOCUS && defocus.aperture != 0.0f;
            const bool blurred = moving || defocused;
            if (blurred) {
                // Jp = K[:2,:2] D P, the expression of the backward's d uv / d pc
                float A0 = Kc[0], A1 = Kc[1], A3 = Kc[3], A4 = Kc[4];
                if (LENS != GSB_LENS_PINHOLE) {
                    A0 = Kc[0] * D[0] + Kc[1] * D[2]; A1 = Kc[0] * D[1] + Kc[1] * D[3];
                    A3 = Kc[3] * D[0] + Kc[4] * D[2]; A4 = Kc[3] * D[1] + Kc[4] * D[3];
                }
                float b00 = 0.0f, b01 = 0.0f, b11 = 0.0f;
                if (moving) {
                    const float iz = 1.0f / pc[2], iz2 = iz * iz;
                    const float dj[6] = {A0 * iz, A1 * iz, (-A0 * pc[0] - A1 * pc[1]) * iz2,
                                         A3 * iz, A4 * iz, (-A3 * pc[0] - A4 * pc[1]) * iz2};
                    float d0, d1;
                    motion_blur_velocity(dj, pc, blur.motion, d0, d1);
                    b00 = (d0 * d0) / 12.0f; b01 = (d0 * d1) / 12.0f; b11 = (d1 * d1) / 12.0f;
                }
                if (defocused) {  // + beta M M^T, M = (A0 A1; A3 A4)
                    const float beta = defocus_variance(defocus, pc[2]);
                    b00 += beta * (A0 * A0 + A1 * A1);
                    b01 += beta * (A0 * A3 + A1 * A4);
                    b11 += beta * (A3 * A3 + A4 * A4);
                }
                c00 += b00; c01 += b01; c10 += b01; c11 += b11;
                cov[0] += b00; cov[1] += b01; cov[2] += b01; cov[3] += b11;  // the radius below: Sigma' + B
                const float det_b = c00 * c11 - c01 * c10;
                blur_c = sqrtf(det / det_b);  // in (0, 1]: B is positive semi-definite
                det = det_b;
            }
            const float inv_det = 1.0f / det;
            // GPCR:311-315 radius from the un-blurred covariance (with BLUR: from Sigma' + B)
            const float ca = cov[0], cd = cov[3];
            const float large = (ca + cd + sqrtf((ca - cd) * (ca - cd) + 4.0f * cov[1] * cov[2])) / 2.0f;
            const float radius = sqrtf(large) * 3.0f;
            // GPCR:299-310 opacity + SH colour along (xyz - camera centre)
            const float opacity = 1.0f / (1.0f + exp_cr(-f[3]));
            // ORTHO: along the camera's forward axis, row 2 of W, the same for every point
            float dx = ORTHO ? T[8] : x - __ldg(&pb->centre[0]), dy = ORTHO ? T[9] : y - __ldg(&pb->centre[1]),
                  dz = ORTHO ? T[10] : z - __ldg(&pb->centre[2]);
            float dn = sqrtf(dx * dx + dy * dy + dz * dz);
            float dinv = 1.0f / dn;
            dx = dinv * dx; dy = dinv * dy; dz = dinv * dz;
            dir0 = dx; dir1 = dy; dir2 = dz;
            bounding_box(u, v, radius, p.W, p.H, min_tu, max_tu, min_tv, max_tv);
            if (EQUIRECT) equirect_columns(u, radius, p.W, min_tu, max_tu);
            ntiles = (max_tu - min_tu) * (max_tv - min_tv);
            // reach-test parameters of this splat; the (tile, splat) tests themselves are done cooperatively by
            // the warp below (one lane per PAIR, not per splat)
            const float rescale_c = FILTER ? rescale * filter_c : blurred ? rescale * blur_c : rescale;
            reach = make_splat_reach(inv_det * c11, inv_det * (-c01), inv_det * c00, rescale_c * opacity);
            if (!p.filter_tiles) reach.mode = 2;
            r0 = make_float4(u, v, inv_det * c11, inv_det * (-c01));
            r1 = make_float4(inv_det * c00, rescale_c, opacity, EQUIRECT ? depth : pc[2]);
            r2.w = radius;
        }
    }

    // ---- warp-cooperative reach filter.  Of the tiles in the reference's 3-sigma square only those where alpha can
    // reach 1/255 on some pixel centre get a sort key (conservative test, common.cuh): a dropped (tile, splat)
    // pair is one the blend would skip on all 256 pixels, so no output changes, and ~1/3 of the pairs go away.
    // The warp's pairs (first 64 tiles of each of its 32 splats) are dealt round-robin to the lanes, so one large
    // splat does not stall the other 31 lanes.
    WarpStage &st = s_stage[warp];
    {
        const int ntv = max_tv - min_tv;
        const int mode = in ? reach.mode : 0;
        st.u[lane] = r0.x; st.v[lane] = r0.y;
        st.a[lane] = reach.a; st.b2[lane] = reach.b2; st.c[lane] = reach.c;
        st.nb_ic[lane] = reach.nb_ic; st.nb_ia[lane] = reach.nb_ia; st.t2[lane] = reach.t2;
        st.min_tu[lane] = min_tu; st.min_tv[lane] = min_tv; st.ntv[lane] = ntv > 0 ? ntv : 1;
        // mode 2 (keep everything): all of the first 64 bits set; mode 0 (never visible): none
        const int n64 = ntiles < 64 ? ntiles : 64;
        const unsigned long long all64 = n64 >= 64 ? ~0ull : ((1ull << n64) - 1ull);
        st.mask_lo[lane] = mode == 2 ? (unsigned int)all64 : 0u;
        st.mask_hi[lane] = mode == 2 ? (unsigned int)(all64 >> 32) : 0u;
        const int tcap = mode == 1 ? n64 : 0;
        int incl_t = tcap;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int o = __shfl_up_sync(0xffffffffu, incl_t, d);
            if (lane >= d) incl_t += o;
        }
        st.pref[lane + 1] = incl_t;
        if (lane == 0) st.pref[0] = 0;
        __syncwarp();
        const int total = st.pref[32];
        for (int q = lane; q < total; q += 32) {
            int lo = 0;  // largest owner with pref[owner] <= q
#pragma unroll
            for (int step = 16; step > 0; step >>= 1)
                if (st.pref[lo + step] <= q) lo += step;
            const int idx = q - st.pref[lo];
            const int ntv_o = st.ntv[lo];
            const int du = idx / ntv_o;
            const int tu = st.min_tu[lo] + du, tv = st.min_tv[lo] + (idx - du * ntv_o);
            SplatReach r;
            r.a = st.a[lo]; r.b2 = st.b2[lo]; r.c = st.c[lo];
            r.nb_ic = st.nb_ic[lo]; r.nb_ia = st.nb_ia[lo]; r.t2 = st.t2[lo];
            r.mode = 1;
            if (tile_reachable(r, st.u[lo], st.v[lo], tu, tv))
                atomicOr(idx < 32 ? &st.mask_lo[lo] : &st.mask_hi[lo], 1u << (idx & 31));
        }
        __syncwarp();
        if (in) {
            const int beyond = ntiles > 64 ? ntiles - 64 : 0;  // tiles past the 64-bit mask are kept untested
            nkeys = mode == 0 ? 0 : __popc(st.mask_lo[lane]) + __popc(st.mask_hi[lane]) + beyond;
        }
    }

    // ---- block-level exclusive scan of the packed pair (count << 36 | tiles)
    const unsigned long long mine = ((unsigned long long)(in ? 1 : 0) << CNT_SHIFT) | (unsigned long long)nkeys;
    unsigned long long incl = mine;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        unsigned long long o = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += o;
    }
    if (lane == 31) s_warp_sums[warp] = incl;
    __syncthreads();
    unsigned long long warp_prefix = 0, block_total = 0;
#pragma unroll
    for (int w = 0; w < SCAN_BLOCK_THREADS / 32; ++w) {
        unsigned long long s = s_warp_sums[w];
        if (w < warp) warp_prefix += s;
        block_total += s;
    }
    // ---- decoupled look-back across blocks: publish first ...
    if (warp == 0 && lane == 0)
        st_state(&p.scan_state[blk], (blk == 0 ? ST_INCLUSIVE : ST_AGGREGATE) | block_total);
    // ---- SH colour (GPCR:299-310), deliberately placed AFTER this block's aggregate is published: the 192 B of
    // coefficients per point are the longest-latency loads of the kernel and nothing upstream of the scan needs
    // the colour, so successor blocks' look-back no longer waits for them, and this block's own look-back
    // overlaps with them.
    if (in) {
        const float4 *frow = reinterpret_cast<const float4 *>(p.features + (size_t)GSB_FEATURE_DIM * i);
                    float sh[16];
                    sh[0] = 0.28209479177387814f;
                    sh[1] = -0.48860251190291987f * dir1;
                    sh[2] = 0.48860251190291987f * dir2;
                    sh[3] = -0.48860251190291987f * dir0;
                    sh[4] = 1.0925484305920792f * dir0 * dir1;
                    sh[5] = -1.0925484305920792f * dir1 * dir2;
                    sh[6] = 0.94617469575755997f * dir2 * dir2 - 0.31539156525251999f;
                    sh[7] = -1.0925484305920792f * dir0 * dir2;
                    sh[8] = 0.54627421529603959f * dir0 * dir0 - 0.54627421529603959f * dir1 * dir1;
                    sh[9] = 0.59004358992664352f * dir1 * (-3.0f * dir0 * dir0 + dir1 * dir1);
                    sh[10] = 2.8906114426405538f * dir0 * dir1 * dir2;
                    sh[11] = 0.45704579946446572f * dir1 * (1.0f - 5.0f * dir2 * dir2);
                    sh[12] = 0.3731763325901154f * dir2 * (5.0f * dir2 * dir2 - 3.0f);
                    sh[13] = 0.45704579946446572f * dir0 * (1.0f - 5.0f * dir2 * dir2);
                    sh[14] = 1.4453057213202769f * dir2 * (dir0 * dir0 - dir1 * dir1);
                    sh[15] = 0.59004358992664352f * dir0 * (-dir0 * dir0 + 3.0f * dir1 * dir1);
                    // SH coefficients are streamed 16 B at a time right where they are consumed (keeps ~50 registers
                    // free; the dot product order k = 0..15 is the oracle's)
                    float col[3];
        #pragma unroll
                    for (int ch = 0; ch < 3; ++ch) {
                        float acc = 0.0f;
        #pragma unroll
                        for (int k4 = 0; k4 < 4; ++k4) {
                            const float4 c4 = __ldg(frow + 2 + 4 * ch + k4);
                            if (k4 == 0) acc = c4.x * sh[0];
                            else acc = acc + c4.x * sh[4 * k4];
                            acc = acc + c4.y * sh[4 * k4 + 1];
                            acc = acc + c4.z * sh[4 * k4 + 2];
                            acc = acc + c4.w * sh[4 * k4 + 3];
                        }
                        col[ch] = sigmoid_cr(acc);
                    }
        r2.x = col[0]; r2.y = col[1]; r2.z = col[2];
    }
    // ---- ... then walk back over the predecessors (warp 0)
    if (warp == 0) {
        unsigned long long exclusive = 0;
        if (blk != 0) {
            int look = blk - 1;
            while (true) {
                const int idx = look - lane;
                unsigned long long word = ST_INCLUSIVE;  // virtual predecessor of block 0
                if (idx >= 0) {
                    word = ld_state(&p.scan_state[idx]);
                    while ((word >> 62) == 0) word = ld_state(&p.scan_state[idx]);
                }
                const unsigned incl_mask = __ballot_sync(0xffffffffu, (word >> 62) == 2);
                unsigned long long val = word & ST_VALUE_MASK;
                if (incl_mask) {
                    const int first = __ffs(incl_mask) - 1;
                    if (lane > first) val = 0;
                    exclusive += warp_sum_u64(val);
                    break;
                }
                exclusive += warp_sum_u64(val);
                look -= 32;
            }
            if (lane == 0) st_state(&p.scan_state[blk], ST_INCLUSIVE | (exclusive + block_total));
        }
        if (lane == 0) {
            s_block_exclusive = exclusive;
            if (blk == p.num_blocks - 1) {
                const unsigned long long tot = exclusive + block_total;
                const long long Ktot = (long long)(tot & ((1ull << CNT_SHIFT) - 1));
                p.counters[CNT_M] = (long long)(tot >> CNT_SHIFT);
                p.counters[CNT_K] = Ktot;
                p.counters[CNT_OVERFLOW] = Ktot > p.key_capacity ? 1 : 0;
            }
        }
    }
    __syncthreads();
    const unsigned long long excl = s_block_exclusive + warp_prefix + (incl - mine);
    const long long off = (long long)(excl >> CNT_SHIFT);
    const long long key_base = (long long)(excl & ((1ull << CNT_SHIFT) - 1));
    if (i < p.N) p.point_offset[i] = in ? (int)off : -1;
    if (ROLLING && i < p.N) rs.row_time[i] = in ? tau : 0.0f;
    if (in) {
        p.point_id[off] = (int)i;
        p.num_tiles[off] = ntiles;
        p.records[3 * off] = r0;
        p.records[3 * off + 1] = r1;
        p.records[3 * off + 2] = r2;
        p.point_in_camera[3 * off] = pc[0];
        p.point_in_camera[3 * off + 1] = pc[1];
        p.point_in_camera[3 * off + 2] = pc[2];
    }

    // ---- warp-cooperative key emission.  GPCR:158-170: key = tile_id << depth_bits | int32(depth * scale), tiles in
    // (tile_u outer, tile_v inner) order.  The key ranges of the warp's splats are adjacent (prefix sum), so
    // dealing the keys round-robin to the lanes makes the stores contiguous and the work balanced.
    {
        const int depth_key = (int)((EQUIRECT ? depth : pc[2]) * p.depth_scale);
        st.depth_key[lane] = depth_key;
        {   // largest depth key of the frame -> CNT_MAX_DEPTH_KEY: the sort runs only the passes its live bits need
            int wmax = in ? depth_key : 0;
#pragma unroll
            for (int d = 16; d > 0; d >>= 1) wmax = max(wmax, __shfl_xor_sync(0xffffffffu, wmax, d));
            int *const slot = reinterpret_cast<int *>(p.counters + CNT_MAX_DEPTH_KEY);
            if (lane == 0 && wmax > *reinterpret_cast<volatile int *>(slot)) atomicMax(slot, wmax);
        }
        st.off[lane] = (int)off;
        st.key_base[lane] = key_base;
        int incl_k = in ? nkeys : 0;
        const int mine_k = incl_k;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int o = __shfl_up_sync(0xffffffffu, incl_k, d);
            if (lane >= d) incl_k += o;
        }
        __syncwarp();  // every lane has finished reading pref[] of the filter phase
        st.pref[lane + 1] = incl_k;
        if (lane == 0) st.pref[0] = 0;
        st.nk64[lane] = in ? mine_k - (ntiles > 64 ? ntiles - 64 : 0) : 0;  // kept tiles among the first 64
        __syncwarp();
        const int total = st.pref[32];
        KeyT *keys = reinterpret_cast<KeyT *>(p.keys);
        const int tiles_x = p.W / GSB_TILE_WIDTH;
        for (int q = lane; q < total; q += 32) {
            int lo = 0;
#pragma unroll
            for (int step = 16; step > 0; step >>= 1)
                if (st.pref[lo + step] <= q) lo += step;
            const int j = q - st.pref[lo];  // j-th kept tile of splat `lo`
            int idx;
            const int nk64 = st.nk64[lo];
            if (j < nk64) {
                const unsigned int mlo = st.mask_lo[lo];
                const int plo = __popc(mlo);
                idx = j < plo ? select_bit32(mlo, j) : 32 + select_bit32(st.mask_hi[lo], j - plo);
            } else {
                idx = 64 + (j - nk64);
            }
            const int ntv_o = st.ntv[lo];
            const int du = idx / ntv_o;
            const int tu = st.min_tu[lo] + du, tv = st.min_tv[lo] + (idx - du * ntv_o);
            const long long pos = st.key_base[lo] + j;
            if (pos < p.key_store_limit) {
                const KeyT tile = EQUIRECT ? (KeyT)((tu % tiles_x + tiles_x) % tiles_x + tv * tiles_x) : (KeyT)(tu + tv * tiles_x);
                keys[pos] = (tile << p.depth_bits) | (KeyT)(unsigned int)st.depth_key[lo];
                p.vals[pos] = st.off[lo];
            }
        }
    }
}

template <typename KeyT>
__global__ void __launch_bounds__(SCAN_BLOCK_THREADS, GSB_PRE_MIN_BLOCKS)
preprocess_kernel(const PreParams p) {
    preprocess_body<KeyT, GSB_LENS_PINHOLE>(p, LensParams());
}

// The parameter block of the lens instantiations: the default kernel keeps PreParams as it is.
struct PreLensParams : PreParams {
    LensParams lens;
};

template <typename KeyT, int LENS>
__global__ void __launch_bounds__(SCAN_BLOCK_THREADS, GSB_PRE_MIN_BLOCKS)
preprocess_lens_kernel(const PreLensParams p) {
    preprocess_body<KeyT, LENS>(p, p.lens);
}

// The parameter block of the rolling-shutter instantiations (LENS = GSB_LENS_PINHOLE ignores `lens`).
struct PreRsParams : PreLensParams {
    RsParams rs;
};

template <typename KeyT, int LENS>
__global__ void __launch_bounds__(SCAN_BLOCK_THREADS, GSB_PRE_MIN_BLOCKS)
preprocess_rs_kernel(const PreRsParams p) {
    preprocess_body<KeyT, LENS, true>(p, p.lens, p.rs);
}

// The parameter blocks of the FILTER instantiations (the other kernels keep theirs as they are).  The lens block's
// LENS = GSB_LENS_PINHOLE instantiation ignores `lens`.
struct PreFilterParams : PreLensParams {
    const float *filter3d;
};
struct PreRsFilterParams : PreRsParams {
    const float *filter3d;
};

template <typename KeyT, int LENS>
__global__ void __launch_bounds__(SCAN_BLOCK_THREADS, GSB_PRE_MIN_BLOCKS)
preprocess_filter_kernel(const PreFilterParams p) {
    preprocess_body<KeyT, LENS, false, true>(p, p.lens, RsParams(), p.filter3d);
}

template <typename KeyT, int LENS>
__global__ void __launch_bounds__(SCAN_BLOCK_THREADS, GSB_PRE_MIN_BLOCKS)
preprocess_rs_filter_kernel(const PreRsFilterParams p) {
    preprocess_body<KeyT, LENS, true, true>(p, p.lens, p.rs, p.filter3d);
}

// The parameter block of the BLUR instantiations (LENS = GSB_LENS_PINHOLE ignores `lens`, ROLLING = false ignores `rs`).
// DEFOCUS = false ignores `defocus`.
struct PreBlurParams : PreRsParams {
    BlurParams blur;
    DefocusParams defocus;
};

template <typename KeyT, int LENS, bool ROLLING, bool DEFOCUS = false>
__global__ void __launch_bounds__(SCAN_BLOCK_THREADS, GSB_PRE_MIN_BLOCKS)
preprocess_blur_kernel(const PreBlurParams p) {
    preprocess_body<KeyT, LENS, ROLLING, false, true, DEFOCUS>(p, p.lens, p.rs, nullptr, p.blur, p.defocus);
}

template <typename KeyT>
__global__ void __launch_bounds__(SCAN_BLOCK_THREADS, GSB_PRE_MIN_BLOCKS)
preprocess_equirect_kernel(const PreParams p) {
    preprocess_body<KeyT, LENS_EQUIRECT>(p, LensParams());
}

// FILTER = false ignores p.filter3d
template <typename KeyT, bool FILTER>
__global__ void __launch_bounds__(SCAN_BLOCK_THREADS, GSB_PRE_MIN_BLOCKS)
preprocess_ortho_kernel(const PreFilterParams p) {
    preprocess_body<KeyT, LENS_ORTHO, false, FILTER>(p, p.lens, RsParams(), p.filter3d);
}

#ifndef GSB_HOST_EMU  // tests/simt compiles the kernels above as host C++ under the SIMT emulator
// The pose blocks of n (q, t) pairs without clearing anything (gsb200_filter3d_from_views: one per view and object).
int launch_pose_blocks(const float *q_pc, const float *t_pc, int n, PoseBlock *poses, cudaStream_t stream) {
    if (n <= 0) return GSB_OK;
    pose_kernel<<<(n + 63) / 64, 64, 0, stream>>>(q_pc, t_pc, n, poses);
    GSB_CUDA_CHECK(cudaGetLastError());
    return GSB_OK;
}

template <typename KeyT>
static void launch_filter_kernel(int model, bool rolling, dim3 grid, dim3 block, cudaStream_t stream,
                                 const PreRsFilterParams &pr) {
    if (rolling) {
        if (model == GSB_LENS_FISHEYE) preprocess_rs_filter_kernel<KeyT, GSB_LENS_FISHEYE><<<grid, block, 0, stream>>>(pr);
        else if (model == GSB_LENS_OPENCV) preprocess_rs_filter_kernel<KeyT, GSB_LENS_OPENCV><<<grid, block, 0, stream>>>(pr);
        else preprocess_rs_filter_kernel<KeyT, GSB_LENS_PINHOLE><<<grid, block, 0, stream>>>(pr);
        return;
    }
    PreFilterParams pf;
    static_cast<PreLensParams &>(pf) = static_cast<const PreLensParams &>(pr);
    pf.filter3d = pr.filter3d;
    if (model == GSB_LENS_FISHEYE) preprocess_filter_kernel<KeyT, GSB_LENS_FISHEYE><<<grid, block, 0, stream>>>(pf);
    else if (model == GSB_LENS_OPENCV) preprocess_filter_kernel<KeyT, GSB_LENS_OPENCV><<<grid, block, 0, stream>>>(pf);
    else preprocess_filter_kernel<KeyT, GSB_LENS_PINHOLE><<<grid, block, 0, stream>>>(pf);
}

template <typename KeyT, bool DEFOCUS>
static void launch_blur_kernel(int model, bool rolling, dim3 grid, dim3 block, cudaStream_t stream, const PreBlurParams &pb) {
    if (rolling) {
        if (model == GSB_LENS_FISHEYE) preprocess_blur_kernel<KeyT, GSB_LENS_FISHEYE, true, DEFOCUS><<<grid, block, 0, stream>>>(pb);
        else if (model == GSB_LENS_OPENCV) preprocess_blur_kernel<KeyT, GSB_LENS_OPENCV, true, DEFOCUS><<<grid, block, 0, stream>>>(pb);
        else preprocess_blur_kernel<KeyT, GSB_LENS_PINHOLE, true, DEFOCUS><<<grid, block, 0, stream>>>(pb);
    } else {
        if (model == GSB_LENS_FISHEYE) preprocess_blur_kernel<KeyT, GSB_LENS_FISHEYE, false, DEFOCUS><<<grid, block, 0, stream>>>(pb);
        else if (model == GSB_LENS_OPENCV) preprocess_blur_kernel<KeyT, GSB_LENS_OPENCV, false, DEFOCUS><<<grid, block, 0, stream>>>(pb);
        else preprocess_blur_kernel<KeyT, GSB_LENS_PINHOLE, false, DEFOCUS><<<grid, block, 0, stream>>>(pb);
    }
}

int launch_preprocess(const GsbForwardArgs &a, const Workspace &ws, cudaStream_t stream, const LensParams *lens,
                      const RsParams *rs, const float *filter3d, const BlurParams *blur, const DefocusParams *defocus) {
    const GsbWorkspaceLayout &L = ws.layout;
    {
        // per-frame state to zero: [counters, sort_state) and [tile_start, zero_bytes) -- every offset is 256-B aligned
        const int clear0_vec = (int)((L.sort_state - L.counters) / 16), clear1_vec = (int)((L.zero_bytes - L.tile_start) / 16);
        const int threads = 64;
        const int pose_blocks = (a.num_objects + threads - 1) / threads;
        int clear_blocks = (clear0_vec + clear1_vec + 4 * threads - 1) / (4 * threads);  // four 16-B stores per thread
        if (clear_blocks > 4 * num_sms()) clear_blocks = 4 * num_sms();
        const int blocks = pose_blocks > clear_blocks ? pose_blocks : clear_blocks;
        pose_kernel<<<blocks > 0 ? blocks : 1, threads, 0, stream>>>(
            a.q_pointcloud_camera, a.t_pointcloud_camera, a.num_objects, ws.poses,
            reinterpret_cast<uint4 *>(ws.counters), clear0_vec, reinterpret_cast<uint4 *>(ws.tile_start), clear1_vec);
        GSB_CUDA_CHECK(cudaGetLastError());
    }
    if (a.num_points <= 0) return GSB_OK;
    PreParams p;
    p.N = a.num_points;
    p.xyz = a.pointcloud;
    p.features = a.pointcloud_features;
    p.invalid = reinterpret_cast<const signed char *>(a.point_invalid_mask);
    p.obj_id = a.point_object_id;
    p.poses = ws.poses;
    p.K = a.camera_intrinsics;
    p.W = a.camera_width;
    p.H = a.camera_height;
    p.near_plane = a.near_plane;
    p.far_plane = a.far_plane;
    p.depth_scale = a.depth_to_sort_key_scale;
    p.depth_bits = L.depth_bits;
    p.skip_q_normalise = (a.flags & GSB_FLAG_Q_ALREADY_NORMALISED) ? 1 : 0;
    p.filter_tiles = (a.flags & GSB_FLAG_KEEP_ALL_TILE_PAIRS) ? 0 : 1;
    p.key_capacity = a.key_capacity;
    p.key_store_limit = ws.layout.key_capacity_padded;
    p.num_blocks = L.scan_blocks;
    p.counters = ws.counters;
    p.tickets = ws.tickets;
    p.scan_state = ws.scan_state;
    p.point_id = ws.point_id;
    p.point_offset = ws.point_offset;
    p.num_tiles = ws.num_tiles;
    p.records = ws.records;
    p.point_in_camera = ws.point_in_camera;
    p.keys = ws.keys_a;
    p.vals = ws.vals_a;
    if (lens != nullptr && lens->model == LENS_ORTHO) {  // gsb200_forward_ortho: the 3D filter or no other extension
        PreFilterParams pf;
        static_cast<PreParams &>(pf) = p;
        pf.lens = *lens;
        pf.filter3d = filter3d;
        const dim3 grid(L.scan_blocks), block(SCAN_BLOCK_THREADS);
        if (L.key_bytes == 4) {
            if (filter3d != nullptr) preprocess_ortho_kernel<unsigned int, true><<<grid, block, 0, stream>>>(pf);
            else preprocess_ortho_kernel<unsigned int, false><<<grid, block, 0, stream>>>(pf);
        } else {
            if (filter3d != nullptr) preprocess_ortho_kernel<unsigned long long, true><<<grid, block, 0, stream>>>(pf);
            else preprocess_ortho_kernel<unsigned long long, false><<<grid, block, 0, stream>>>(pf);
        }
    } else if (blur != nullptr || defocus != nullptr) {
        PreBlurParams pb;
        static_cast<PreParams &>(pb) = p;
        pb.lens = lens != nullptr ? *lens : LensParams();
        pb.rs = rs != nullptr ? *rs : RsParams();
        pb.blur = blur != nullptr ? *blur : BlurParams{};  // zero motion: the defocus alone
        pb.defocus = defocus != nullptr ? *defocus : DefocusParams();
        const int model = lens != nullptr ? lens->model : GSB_LENS_PINHOLE;
        const dim3 grid(L.scan_blocks), block(SCAN_BLOCK_THREADS);
        const bool r = rs != nullptr;
        if (defocus != nullptr) {
            if (L.key_bytes == 4) launch_blur_kernel<unsigned int, true>(model, r, grid, block, stream, pb);
            else launch_blur_kernel<unsigned long long, true>(model, r, grid, block, stream, pb);
        } else {
            if (L.key_bytes == 4) launch_blur_kernel<unsigned int, false>(model, r, grid, block, stream, pb);
            else launch_blur_kernel<unsigned long long, false>(model, r, grid, block, stream, pb);
        }
    } else if (filter3d != nullptr) {
        PreRsFilterParams pr;
        static_cast<PreParams &>(pr) = p;
        pr.lens = lens != nullptr ? *lens : LensParams();
        pr.rs = rs != nullptr ? *rs : RsParams();
        pr.filter3d = filter3d;
        const int model = lens != nullptr ? lens->model : GSB_LENS_PINHOLE;
        const dim3 grid(L.scan_blocks), block(SCAN_BLOCK_THREADS);
        if (L.key_bytes == 4) launch_filter_kernel<unsigned int>(model, rs != nullptr, grid, block, stream, pr);
        else launch_filter_kernel<unsigned long long>(model, rs != nullptr, grid, block, stream, pr);
    } else if (rs != nullptr) {
        PreRsParams pr;
        static_cast<PreParams &>(pr) = p;
        pr.lens = lens != nullptr ? *lens : LensParams();
        pr.rs = *rs;
        const int model = lens != nullptr ? lens->model : GSB_LENS_PINHOLE;
        const dim3 grid(L.scan_blocks), block(SCAN_BLOCK_THREADS);
        if (L.key_bytes == 4) {
            if (model == GSB_LENS_FISHEYE) preprocess_rs_kernel<unsigned int, GSB_LENS_FISHEYE><<<grid, block, 0, stream>>>(pr);
            else if (model == GSB_LENS_OPENCV) preprocess_rs_kernel<unsigned int, GSB_LENS_OPENCV><<<grid, block, 0, stream>>>(pr);
            else preprocess_rs_kernel<unsigned int, GSB_LENS_PINHOLE><<<grid, block, 0, stream>>>(pr);
        } else {
            if (model == GSB_LENS_FISHEYE) preprocess_rs_kernel<unsigned long long, GSB_LENS_FISHEYE><<<grid, block, 0, stream>>>(pr);
            else if (model == GSB_LENS_OPENCV) preprocess_rs_kernel<unsigned long long, GSB_LENS_OPENCV><<<grid, block, 0, stream>>>(pr);
            else preprocess_rs_kernel<unsigned long long, GSB_LENS_PINHOLE><<<grid, block, 0, stream>>>(pr);
        }
    } else if (lens != nullptr && lens->model == LENS_EQUIRECT) {  // gsb200_forward_equirect: no other extension
        if (L.key_bytes == 4) preprocess_equirect_kernel<unsigned int><<<L.scan_blocks, SCAN_BLOCK_THREADS, 0, stream>>>(p);
        else preprocess_equirect_kernel<unsigned long long><<<L.scan_blocks, SCAN_BLOCK_THREADS, 0, stream>>>(p);
    } else if (lens != nullptr) {
        PreLensParams pl;
        static_cast<PreParams &>(pl) = p;
        pl.lens = *lens;
        const bool fisheye = lens->model == GSB_LENS_FISHEYE;
        if (L.key_bytes == 4) {
            if (fisheye) preprocess_lens_kernel<unsigned int, GSB_LENS_FISHEYE><<<L.scan_blocks, SCAN_BLOCK_THREADS, 0, stream>>>(pl);
            else preprocess_lens_kernel<unsigned int, GSB_LENS_OPENCV><<<L.scan_blocks, SCAN_BLOCK_THREADS, 0, stream>>>(pl);
        } else {
            if (fisheye)
                preprocess_lens_kernel<unsigned long long, GSB_LENS_FISHEYE><<<L.scan_blocks, SCAN_BLOCK_THREADS, 0, stream>>>(pl);
            else
                preprocess_lens_kernel<unsigned long long, GSB_LENS_OPENCV><<<L.scan_blocks, SCAN_BLOCK_THREADS, 0, stream>>>(pl);
        }
    } else if (L.key_bytes == 4)
        preprocess_kernel<unsigned int><<<L.scan_blocks, SCAN_BLOCK_THREADS, 0, stream>>>(p);
    else
        preprocess_kernel<unsigned long long><<<L.scan_blocks, SCAN_BLOCK_THREADS, 0, stream>>>(p);
    GSB_CUDA_CHECK(cudaGetLastError());
    return GSB_OK;
}
#endif  // GSB_HOST_EMU

}  // namespace gsb
