// blend_bwd_transposed.cu -- loop A of the backward (GPCR:531-705); the DEFAULT implementation (the butterfly kernel of
// blend_bwd.cu stays selectable: backward_impl="butterfly").  Verified on the CPU under tests/simt (the kernel body compiled as host C++ and run by a
// lock-step SIMT emulator against the butterfly kernel and the oracle) and on the GPU by every backward parity test.
//
// blend_bwd.cu reduces the 11 per-splat partials of every (warp, splat) visit across the 32 pixels of the warp with a
// 13-shuffle butterfly: ~52 of the ~117 SASS instructions of a visit.  Here a warp copies the splats of its culled list,
// TB_CHUNK at a time, into a private chunk buffer (a partial chunk at the end of a staging batch is carried over and topped
// up from the next batch, so only the last chunk of a tile can be short) and works on a chunk in two phases:
//   phase 1 (lane = pixel, as before): the sequential part of GPCR:609-657 -- alpha, the transmittance recursion and
//     the colour recursion -- which leaves two numbers per (pixel, splat): G = dL/dalpha * alpha and alpha*T.  They go
//     as one float2 to a 32 x TB_CHUNK exchange buffer in shared memory (bank arithmetic at TbShared);
//   phase 2 (lane = splat; 32/TB_CHUNK lanes share a splat, each takes TB_CHUNK/8 rows of the 8 x 4 patch): along a row
//     conic*d is linear in the pixel's column offset k, so a lane sums only G, k G and k^2 G per row and rebuilds the five
//     geometric partials from these moments after the row; the colour partials are summed per pixel.  The lanes of a
//     splat are added with log2(32/TB_CHUNK) shuffles per value, and the TB_CHUNK finished rows leave through shared
//     memory as 16-byte vector REDs, 3 per row (same 2 sectors per (warp, splat) as the butterfly kernel).
// STATS = false (GSB_FLAG_NO_HOOK_STATS, the reference's need_extra_info = False, GPCR:521, 690-704) drops the |d/duv|
// magnitude, the affected-pixel count and the per-pixel magnitude image.
// DEPTH = true (gsb200_backward_with_depth; the reference never differentiates its depth output) adds the gradient of the
// depth map D = sum w z / S (S = sum w = the accumulated alpha).  With g^ = dL/dD / S per pixel:
//   through alpha: D behaves like a colour channel whose "colour" is z - D, weighted by g^ -- phase 1 folds it into the
//     colour recursion (fast path: cg += g^ z - g^ D; exact path: a fourth accumulator w3 = sum (z - D) alpha T);
//   direct:        dD/dz_i = alpha_i T_i / S -- phase 2 sums alpha T g^ per splat into the spare word 11 of the
//     accumulator row (g^ rides in the unused .w of the warp's dL/dimage copy), which backward_points_kernel<_, true>
//     turns into dL/dxyz along the camera's viewing axis.
// ALPHA = true (gsb200_backward_aux with an alpha gradient) adds the gradient of the accumulated alpha S = 1 - prod (1 - alpha).
// S is the blend of a colour channel whose colour is 1, so dS/dalpha_i = T_i - sum_{j behind i} w_j / (1 - alpha_i)
// = T_final / (1 - alpha_i), and with g_S = dL/dS per pixel (a register of phase 1; no direct term, nothing in phase 2):
//   fast path:  the one-scalar recursion's cg = sum g c_i becomes sum g c_i + g_S (the FMA chain starts at g_S, or at
//     g_S - g^ D with DEPTH);
//   exact path: a_grad += g_S T_final / (1 - alpha) for a contributing pair.
// CF = 4, 8 or 16 (gsb200_backward_ext) adds the gradient of C <= CF per-Gaussian feature channels F_p = sum_i w_i f_i
// (w_i = alpha_i T_i, the image's weights).  Each channel is one more colour channel of the blend; with g_{p,c} = dL/dF_{p,c}:
//   phase 1: s = sum_c g_{p,c} f_{i,c} per visit (the pixel's g in registers, the chunk's feature rows in shared memory)
//     fast path:  cg += s, so the one-scalar recursion carries it to the splats in front and G picks it up;
//     exact path: a fifth accumulator wF = sum_{j behind} s_j alpha_j T_j, a_grad += s T_i - wF / (1 - alpha);
//   phase 2: dL/df_{i,c} = sum_p (alpha T)_{p,i} g_{p,c} from the exchange buffer and the warp's g staged in shared memory,
//     one shuffle level, then RED.ADD (F32x4 where C % 4 == 0) into the (N,C) rows.
// The feature buffers are appended to the dynamic shared-memory image (TbFeat) and the kernel is compiled for 2 CTAs per
// SM (DESIGN section 3); the existing buffers, the accumulator rows and the workspace are unchanged.
// WRAP = true (gsb200_backward_equirect): the panorama's seam, staged as in the forward (equirect_wrap_u, common.cuh): every
// later use of u -- phase 1's d0 and phase 2's row offsets -- sees the copy nearest the tile, and dL/du is unchanged by the shift.
#include <type_traits>

#include "blend_bwd.cuh"

namespace gsb {

// Splats per chunk: 16 (a phase-2 lane owns two rows of the patch; 71 KB, 80 registers -> 3 CTAs per SM) or 8 (one row;
// 52 KB, 64 registers -> 4 CTAs per SM).  On an H100 at C3 the 4th CTA does not pay for the second shuffle level and
// the halved amortisation of the chunk's epilogue: 16 is the faster (DESIGN section 3).
#ifndef GSB_TB_CHUNK
#define GSB_TB_CHUNK 16
#endif
#ifndef GSB_TB_MIN_BLOCKS  // tuning knob (GSB200_DEFINES="-DGSB_TB_CHUNK=8 -DGSB_TB_MIN_BLOCKS=4")
#if GSB_TB_CHUNK == 8
#define GSB_TB_MIN_BLOCKS 4
#else
#define GSB_TB_MIN_BLOCKS 3
#endif
#endif
constexpr int TB_CHUNK = GSB_TB_CHUNK;
static_assert(TB_CHUNK == 8 || TB_CHUNK == 16, "a phase-2 lane takes whole rows of the 8 x 4 patch");
constexpr int TB_ROWS = TB_CHUNK / 8;  // patch rows per phase-2 lane
constexpr int TB_ROW = TB_CHUNK + 1;   // row stride (float2) of the (pixel, splat) exchange buffer: odd, see below

// Exchange buffer bank arithmetic.  A 64-bit shared access is served per half-warp (16 lanes x 8 B = the 32 banks), so
// both patterns take their minimum of 2 wavefronts when the 16 float2 indices of a half-warp are distinct mod 16:
//   phase 1 (lane = pixel p, splat i fixed):  p * TB_ROW + i, TB_ROW odd -> distinct for 16 consecutive p;
//   phase 2 (pixel pp = 8 row + k, k fixed):  TB_CHUNK = 16: one pixel, 16 consecutive splats; TB_CHUNK = 8: splats
//     0..7 of pixels pp and pp + 8, 8 * 9 = 72 = 8 mod 16 apart -> two disjoint runs of 8.
struct TbWarp {  // a warp's private buffers: one base register addresses them all
    float4 g[32];                       // dL/dimage of the warp's pixels
    float4 chunk[3][TB_CHUNK];          // records of the current chunk's splats [plane][slot]; the radius word of plane 2
                                        //   carries the splat's position in the tile's sorted list
    float2 x[32 * TB_ROW];              // (G, alpha * T) per (pixel, splat of the chunk); reused for the finished rows
    int chunk_off[TB_CHUNK];            // accumulator rows of the chunk's splats (-1 after phase 2 if nothing is to be added)
    unsigned char list[GSB_TILE_PIXELS];  // elements of the current batch to visit, back to front
};
struct TbShared {  // dynamic shared memory image: 52 KB (TB_CHUNK = 8) or 71 KB (16)
    float4 rec[2 * 3 * GSB_TILE_PIXELS];  // [buf][plane][splat] as in blend_bwd.cu; the radius word of plane 2 (unused by
                                          //   the backward) carries the splat's in-camera offset
    TbWarp w[8];
    unsigned int bits[2][8][8];           // [buf][consumer warp patch][loader warp]
    float2 origin;                        // the tile's corner in pixels: re-read where needed rather than held in two registers
    int max_last;
};
static_assert(2 * 32 * TB_ROW >= TB_CHUNK * GSB_ACCUM_FLOATS && GSB_ACCUM_FLOATS == 12,
              "the finished rows (3 float4 each) must fit into the exchange buffer");
// the H100 has 228 KB of shared memory per SM and reserves 1 KB of it per resident CTA
static_assert(GSB_TB_MIN_BLOCKS * (sizeof(TbShared) + 1024) <= 228 * 1024,
              "the shared-memory image does not allow GSB_TB_MIN_BLOCKS CTAs per SM");

template <int CF>
struct TbFeat {  // CF > 0: appended to the dynamic shared-memory image after TbShared
    int row[2][GSB_TILE_PIXELS];  // [buf][element]: scene rows of the staged splats
    struct Warp {
        float4 g[32][CF / 4];         // dL/dF of the warp's pixels (zero past C)
        float4 f[TB_CHUNK][CF / 4];   // feature rows of the current chunk's splats (zero past C)
        int row[TB_CHUNK];            // their scene rows
    } w[8];
};
constexpr int TB_FEAT_MIN_BLOCKS = 2;
constexpr int tb_min_blocks(int cf) { return cf == 0 ? GSB_TB_MIN_BLOCKS : TB_FEAT_MIN_BLOCKS; }
template <int CF>
constexpr size_t tb_smem_bytes() { return sizeof(TbShared) + (CF > 0 ? sizeof(TbFeat<(CF > 0 ? CF : 4)>) : 0); }
static_assert(sizeof(TbShared) % 16 == 0, "TbFeat starts 16-byte aligned");
static_assert(TB_FEAT_MIN_BLOCKS * (tb_smem_bytes<16>() + 1024) <= 228 * 1024,
              "the feature instantiations' shared-memory image does not allow TB_FEAT_MIN_BLOCKS CTAs per SM");

#ifdef GSB_HOST_EMU
static inline unsigned char *tb_dynamic_smem() { return simt_emu::dynamic_smem(); }
#else
extern __shared__ __align__(16) unsigned char gsb_tb_dynamic_smem[];
__device__ __forceinline__ unsigned char *tb_dynamic_smem() { return gsb_tb_dynamic_smem; }
#endif

#ifndef GSB_TB_P1_UNROLL
#define GSB_TB_P1_UNROLL 4  // phase-1 splats per loop trip
#endif
constexpr int TB_P1_UNROLL = GSB_TB_P1_UNROLL;
static_assert(TB_CHUNK % TB_P1_UNROLL == 0, "a full chunk is a whole number of phase-1 groups");
// one 16-byte RED.ADD of four f32 (sm_90: atomicAdd on a float4 in global memory); the emulator adds word by word
__device__ __forceinline__ void red_add_f32x4(float *addr, const float4 v) {
#ifdef GSB_HOST_EMU
    atomicAdd(addr, v.x);
    atomicAdd(addr + 1, v.y);
    atomicAdd(addr + 2, v.z);
    atomicAdd(addr + 3, v.w);
#else
    atomicAdd(reinterpret_cast<float4 *>(addr), v);
#endif
}
// P if (idx < last && P >= 1/255) else 0 -- the two tests folded into one predicate (ISETP, FSETP.AND, FSEL instead of
// the two selects the compiler makes of the && expression)
__device__ __forceinline__ float keep_if_contributing(float P, int idx, int last) {
#ifdef GSB_HOST_EMU
    return ((idx < last) && (P >= 1.0f / 255.0f)) ? P : 0.0f;
#else
    float r;
    asm("{\n"
        ".reg .pred p, q;\n"
        "setp.lt.s32 q, %2, %3;\n"
        "setp.ge.and.f32 p, %1, 0f3B808081, q;\n"   // 1.0f / 255.0f
        "selp.f32 %0, %1, 0f00000000, p;\n"
        "}\n"
        : "=f"(r)
        : "f"(P), "r"(idx), "r"(last));
    return r;
#endif
}

template <int CF>
using TbParams = typename std::conditional<CF == 0, BlendBwdParams, BlendBwdFeatParams>::type;

template <bool EXACT_EXP, bool STATS, bool COUNT = false, bool DEPTH = false, bool ALPHA = false, int CF = 0, bool WRAP = false>
__global__ void __launch_bounds__(GSB_TILE_PIXELS, tb_min_blocks(CF))
blend_backward_transposed_kernel(const TbParams<CF> p) {
    static_assert(!(COUNT && (DEPTH || ALPHA || CF)), "the work-counter diagnostic runs the default arithmetic only");
    static_assert(CF % 4 == 0 && CF <= 16, "features: whole float4 groups");
    TbShared &S = *reinterpret_cast<TbShared *>(tb_dynamic_smem());
    constexpr int NV = STATS ? 11 : 9;
    constexpr int CFW = CF > 0 ? CF : 4;
    // phase-1 splats per loop trip: at CF = 16 the group's hoisted feature rows would not fit the 128 registers of 2 CTAs per SM
    constexpr int P1U = CF >= 16 ? 2 : TB_P1_UNROLL;
    TbFeat<CFW> &SF = *reinterpret_cast<TbFeat<CFW> *>(tb_dynamic_smem() + sizeof(TbShared));  // CF > 0 only

    const int tile = blockIdx.x;
    const int tu = tile % p.tiles_x, tv = tile / p.tiles_x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int pu = tu * GSB_TILE_WIDTH + (warp & 1) * 8 + (lane & 7);
    const int pv = tv * GSB_TILE_HEIGHT + (warp >> 1) * 4 + (lane >> 3);
    const float px = (float)pu + 0.5f, py = (float)pv + 0.5f;
    const size_t pix = (size_t)pv * p.W + pu;
    const int start = p.tile_start[tile];

    const int last = p.last_effective[pix];
    float T = 1.0f - p.acc_alpha[pix];  // GPCR:559-560
    float w0 = 0.0f, w1 = 0.0f, w2 = 0.0f;
    const float g0 = p.grad_image[3 * pix], g1 = p.grad_image[3 * pix + 1], g2 = p.grad_image[3 * pix + 2];
    float mag0 = 0.0f, mag1 = 0.0f;
    unsigned int n_visits = 0, n_pairs = 0;  // COUNT only
    // DEPTH only: gd = dL/dD / S (0 where nothing is blended: S = 0 exactly, and then no pair contributes either); hd = gd D
    // on the fast path, D on the exact one.  S >= 1/255 wherever a splat is blended, so the forward's 1e-6 clamp of S
    // never applies to a pixel with something to differentiate.
    float gd = 0.0f, hd = 0.0f, w3 = 0.0f;
    if (DEPTH) {
        const float Sa = p.acc_alpha[pix];
        gd = Sa > 0.0f ? p.grad_depth[pix] / Sa : 0.0f;
        hd = EXACT_EXP ? p.depth[pix] : gd * p.depth[pix];
    }
    // ALPHA only: ga = g_S (- hd with DEPTH) starts the fast path's colour chain; g_S T_final on the exact path
    float ga = 0.0f;
    if (ALPHA) {
        const float gs = p.grad_alpha[pix];
        ga = EXACT_EXP ? gs * T : DEPTH ? gs - hd : gs;
    }
    TbWarp &Wp = S.w[warp];
    Wp.g[lane] = make_float4(g0, g1, g2, gd);
    // CF > 0: this pixel's dL/dF (registers for phase 1, the warp's shared copy for phase 2); wF the exact path's accumulator
    float gf[CFW];
    float wF;
    typename TbFeat<CFW>::Warp &WF = SF.w[warp];
    const BlendFeatureParams fp = feature_params(p);
    const int C = CF > 0 ? fp.channels : 0;
    if constexpr (CF > 0) {
        wF = 0.0f;
        const float *src = fp.grad_feature_map + pix * C;
#pragma unroll
        for (int c = 0; c < CF; ++c) gf[c] = c < C ? src[c] : 0.0f;
#pragma unroll
        for (int c = 0; c < CF; c += 4) WF.g[lane][c / 4] = make_float4(gf[c], gf[c + 1], gf[c + 2], gf[c + 3]);
    }

    // phase-2 role of this lane: splat `ci` of the chunk, rows row0 .. row0 + TB_ROWS - 1 of the patch
    const int ci = lane % TB_CHUNK, row0 = (lane / TB_CHUNK) * TB_ROWS;
    float2 *const x = Wp.x;
    float4 *const fin = reinterpret_cast<float4 *>(x);  // the finished rows: 3 float4 per splat of the chunk
    unsigned char *const list = Wp.list;

    int warp_last = last;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) warp_last = max(warp_last, __shfl_xor_sync(0xffffffffu, warp_last, d));
    if (tid == 0) {
        S.max_last = start;
        S.origin = make_float2((float)(tu * GSB_TILE_WIDTH), (float)(tv * GSB_TILE_HEIGHT));
    }
    __syncthreads();
    if (lane == 0) atomicMax(&S.max_last, warp_last);
    __syncthreads();
    const int end = min(p.tile_end[tile], S.max_last);

    float4 *const ck0 = Wp.chunk[0], *const ck1 = Wp.chunk[1], *const ck2 = Wp.chunk[2];
    int *const ck_off = Wp.chunk_off;
    int have = 0;  // splats waiting in the chunk buffer (warp-uniform)

    // One barrier per staging batch (double-buffered, see blend_fwd.cu).  After the last batch one more trip through the
    // loop (real == false: no staging, no barrier) flushes the short chunk that is left.
    int buf = 0;
    for (int block_end = end;; block_end -= GSB_TILE_PIXELS, buf ^= 1) {
        const bool real = block_end > start;  // CTA-uniform
        int count = 0;
        float4 *const s_r0 = S.rec + buf * 3 * GSB_TILE_PIXELS;
        float4 *const s_r1 = s_r0 + GSB_TILE_PIXELS, *const s_r2 = s_r0 + 2 * GSB_TILE_PIXELS;
        if (real) {
            const int block_start = max(block_end - GSB_TILE_PIXELS, start);
            {
                const int idx = block_end - 1 - tid;  // element j <-> sorted index block_end-1-j
                unsigned int mask = 0;
                if (idx >= block_start) {
                    const int o = __ldg(&p.sorted_vals[idx]);
                    const float4 *rec = p.records + 3 * (size_t)o;
                    float4 r0 = __ldg(rec);
                    const float4 r1 = __ldg(rec + 1);
                    if (WRAP) r0.x = equirect_wrap_u(r0.x, S.origin.x, (float)p.W);
                    if (EXACT_EXP) {
                        s_r0[tid] = r0;
                        s_r1[tid] = r1;
                    } else {  // the forward's staged planes (common.cuh): u v A B | C rescale*opacity 1-opacity depth
                        float4 f0, f1;
                        fast_planes(r0, r1, f0, f1);
                        s_r0[tid] = f0;
                        s_r1[tid] = f1;
                    }
                    float4 r2 = __ldg(rec + 2);
                    r2.w = __int_as_float(o);  // in-camera offset instead of the radius (unused here)
                    s_r2[tid] = r2;
                    if constexpr (CF > 0) SF.row[buf][tid] = __ldg(&fp.point_id[o]);
                    mask = splat_patch_mask(r0.x, r0.y, r0.z, r0.w, r1.x, r1.y * r1.z, S.origin.x, S.origin.y);
                }
#pragma unroll
                for (int w = 0; w < 8; ++w) {
                    const unsigned int bits = __ballot_sync(0xffffffffu, (mask >> w) & 1u);
                    if (lane == 0) S.bits[buf][w][warp] = bits;
                }
            }
            __syncthreads();
            if (tid == 0) GSB_EMU_COUNT(EC_BATCHES, 1);
            if (block_start < warp_last) {  // otherwise every splat of this batch is behind the whole patch (warp-uniform)
                // ordered visit list of this patch: set bits of the 8 words, minus the first `skip` elements of the batch
                // (those lie at or behind the patch's deepest effective splat)
                const int skip = block_end - warp_last;
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    unsigned int bits = S.bits[buf][warp][k];
                    const int lo = skip - 32 * k;
                    if (lo >= 32) bits = 0u;
                    else if (lo > 0) bits &= ~((1u << lo) - 1u);
                    if ((bits >> lane) & 1u)
                        list[count + __popc(bits & ((1u << lane) - 1u))] = (unsigned char)(k * 32 + lane);
                    count += __popc(bits);
                }
                __syncwarp();
            }
        }

        int pos = 0;
#pragma unroll 1
        do {
            if (pos < count) {  // top the chunk buffer up from this batch's list
                const int take = min(TB_CHUNK - have, count - pos);
                if (lane < take) {
                    const int j = list[pos + lane], slot = have + lane;
                    ck0[slot] = s_r0[j];
                    ck1[slot] = s_r1[j];
                    float4 r2 = s_r2[j];
                    ck_off[slot] = __float_as_int(r2.w);
                    r2.w = __int_as_float(block_end - 1 - j);  // sorted index instead of the in-camera offset
                    ck2[slot] = r2;
                    if constexpr (CF > 0) {  // the splat's feature row, zero-padded to CF
                        const int row = SF.row[buf][j];
                        WF.row[slot] = row;
                        const float *src = fp.features + (size_t)row * C;
#pragma unroll
                        for (int c = 0; c < CF; c += 4)
                            WF.f[slot][c / 4] = make_float4(c < C ? __ldg(src + c) : 0.0f, c + 1 < C ? __ldg(src + c + 1) : 0.0f,
                                                            c + 2 < C ? __ldg(src + c + 2) : 0.0f,
                                                            c + 3 < C ? __ldg(src + c + 3) : 0.0f);
                    }
                }
                have += take;
                pos += take;
                __syncwarp();
            }
            if (have == TB_CHUNK || (!real && have > 0)) {
                const int n = have;
                have = 0;
                if (COUNT) n_visits += (lane == 0) ? (unsigned int)n : 0u;
                if (lane == 0) {
                    GSB_EMU_COUNT(EC_TB_SPLATS, n);
                    GSB_EMU_COUNT(EC_TB_CHUNKS, 1);
                }
                // ---- phase 1: lane = pixel; sequential over the chunk's splats (back to front)
                const auto p1 = [&](const int i) -> float2 {
                    const float4 r0 = ck0[i];  // u v a b                   (fast path: u v A B, conic scaled by -log2(e)/2)
                    const float4 r1 = ck1[i];  // c rescale opacity depth   (fast path: C rescale*opacity 1-opacity depth)
                    const float4 r2 = ck2[i];  // r g b | sorted index
                    const int idx = __float_as_int(r2.w);
                    const float d0 = px - r0.x, d1 = py - r0.y;
                    float sf = 0.0f;  // CF > 0: s = sum_c g_c f_c, the feature channels' share of the colour-gradient product
                    if constexpr (CF > 0) {
#pragma unroll
                        for (int c = 0; c < CF; c += 4) {
                            const float4 f = WF.f[i][c / 4];
                            sf = fmaf(gf[c], f.x, sf);
                            sf = fmaf(gf[c + 1], f.y, sf);
                            sf = fmaf(gf[c + 2], f.z, sf);
                            sf = fmaf(gf[c + 3], f.w, sf);
                        }
                    }
                    float G, aT;
                    if (EXACT_EXP) {
                        const float q0 = r0.z * d0 + r0.w * d1;
                        const float q1 = r0.w * d0 + r1.x * d1;
                        const float gp = expf(-0.5f * (d0 * q0 + d1 * q1)) * r1.y;
                        const float prod_alpha = gp * r1.z;
                        const bool contributes = (idx < last) && (prod_alpha >= 1.0f / 255.0f);
                        const float alpha = fminf(prod_alpha, 0.99f);
                        const float inv = 1.0f / (1.0f - alpha);
                        const float Tn = T * inv;
                        aT = contributes ? alpha * Tn : 0.0f;
                        float a_grad = contributes ? (r2.x * Tn - w0 * inv) * g0 + (r2.y * Tn - w1 * inv) * g1 +
                                                         (r2.z * Tn - w2 * inv) * g2
                                                   : 0.0f;
                        if (DEPTH) {  // the depth map's "colour" z - D
                            const float e = r1.w - hd;
                            a_grad += contributes ? (e * Tn - w3 * inv) * gd : 0.0f;
                            w3 = fmaf(e, aT, w3);
                        }
                        if (ALPHA) a_grad += contributes ? ga * inv : 0.0f;  // g_S T_final / (1 - alpha)
                        if constexpr (CF > 0) {  // the feature channels, summed: "colour" times gradient s
                            a_grad += contributes ? sf * Tn - wF * inv : 0.0f;
                            wF = fmaf(sf, aT, wF);
                        }
                        T = contributes ? Tn : T;
                        w0 = fmaf(r2.x, aT, w0);
                        w1 = fmaf(r2.y, aT, w1);
                        w2 = fmaf(r2.z, aT, w2);
                        G = a_grad * r1.z * gp;
                        if (STATS) {
                            mag0 += fabsf(G * q0);
                            mag1 += fabsf(G * q1);
                        }
                    } else {
                        // One-scalar colour recursion (see blend_bwd.cu); alpha is the FORWARD's expression on the forward's
                        // staged values (fast_alpha, common.cuh), so both passes take the 1/255 decision on identical bits.
                        // A pair that does not contribute gets P = 0: then alpha = 0, 1/(1-alpha) = 1, T and w0 keep their
                        // values and G = aT = 0 -- no other select is needed.
                        float P = fast_alpha(d0, d1, r0.z, r0.w, r1.x, r1.y);
                        P = keep_if_contributing(P, idx, last);
                        const float alpha = fminf(P, 0.99f);
                        const float inv = rcp_approx(1.0f - alpha);
                        T *= inv;                 // T_i = T_{i+1} / (1 - alpha), GPCR:640
                        aT = alpha * T;
                        // + g_S with ALPHA: the accumulated alpha as a channel of colour 1
                        float cg = fmaf(r2.z, g2, fmaf(r2.y, g1, ALPHA ? fmaf(r2.x, g0, ga) : r2.x * g0));
                        // + gd (z - D): the depth map as a fourth channel (with ALPHA, ga already holds the - hd)
                        if (DEPTH) cg = ALPHA ? fmaf(gd, r1.w, cg) : fmaf(gd, r1.w, cg) - hd;
                        if constexpr (CF > 0) cg += sf;  // + sum_c g_c f_c: the feature channels
                        const float a_grad = fmaf(cg, T, -(w0 * inv));
                        w0 = fmaf(cg, aT, w0);
                        G = a_grad * P;
                        if (STATS) {  // hook only: |d/duv| on the image needs conic * d  (A d0 + B/2 d1 = -log2(e)/2 q0)
                            const float q0 = (-2.0f / GSB_L2E) * fmaf(r0.z, d0, 0.5f * r0.w * d1);
                            const float q1 = (-2.0f / GSB_L2E) * fmaf(0.5f * r0.w, d0, r1.x * d1);
                            mag0 += fabsf(G * q0);
                            mag1 += fabsf(G * q1);
                        }
                    }
                    if (COUNT) n_pairs += aT > 0.0f ? 1u : 0u;
                    return make_float2(G, aT);
                };
                if (n == TB_CHUNK) {
                    // Groups of TB_P1_UNROLL splats, their exchange stores after the group: the compiler cannot tell the
                    // exchange buffer from the chunk buffer, so a store between two splats would keep the next splat's
                    // loads and alpha (independent of the recursion) from being scheduled under the previous one.
#pragma unroll 1
                    for (int i0 = 0; i0 < TB_CHUNK; i0 += P1U) {
                        float2 ex[P1U];
#pragma unroll
                        for (int u = 0; u < P1U; ++u) ex[u] = p1(i0 + u);
#pragma unroll
                        for (int u = 0; u < P1U; ++u) x[lane * TB_ROW + i0 + u] = ex[u];
                    }
                } else {  // the short last chunk of a tile
#pragma unroll 1
                    for (int i = 0; i < n; ++i) x[lane * TB_ROW + i] = p1(i);
                }
                __syncwarp();

                // ---- phase 2: lane = splat ci of the chunk, over the TB_CHUNK pixels of its rows
                const bool active = ci < n;
                float4 s0 = ck0[active ? ci : 0];
                float4 s1 = ck1[active ? ci : 0];
                if (!EXACT_EXP) {  // back to the conic itself (the chunk holds it scaled by -log2(e)/2 for fast_alpha)
                    s0.z *= -2.0f / GSB_L2E;
                    s0.w *= -1.0f / GSB_L2E;
                    s1.x *= -2.0f / GSB_L2E;
                }
                const float ca = s0.z, cb = s0.w, cc = s1.x;  // conic (a, b, c)
                // this lane's rows: pixel centres pxc + kc, kc = k - 3.5 for the pixels k = 0..7 of a row (half-integers:
                // kc and kc^2 are exact)
                const float2 org = S.origin;
                const float pxc = org.x + (float)((warp & 1) * 8) + 4.0f;
                const float pyb = org.y + (float)((warp >> 1) * 4 + row0) + 0.5f;
                const float dxc = pxc - s0.x;  // d0 at the centre of the row
                float acc[12];  // the accumulator row; word 11 only with DEPTH
#pragma unroll
                for (int k = 0; k < 12; ++k) acc[k] = 0.0f;
                float af[CFW];  // CF > 0: sum alpha T g_c over this lane's pixels = dL/df_c of the splat
                if constexpr (CF > 0) {
#pragma unroll
                    for (int c = 0; c < CF; ++c) af[c] = 0.0f;
                }
                unsigned int nz = 0u;
#pragma unroll
                for (int row = 0; row < TB_ROWS; ++row) {
                    // along the row d0 = dxc + kc, so conic * d = (q0r + a kc, q1r + b kc): the moments m0 = sum G,
                    // m1 = sum kc G, m2 = sum kc^2 G of the row (one FADD and two FFMA per pixel) give all five geometric sums
                    const float d1 = (pyb + (float)row) - s0.y;
                    const float q0r = fmaf(ca, dxc, cb * d1);
                    const float q1r = fmaf(cb, dxc, cc * d1);
                    float m0 = 0.0f, m1 = 0.0f, m2 = 0.0f;
#pragma unroll
                    for (int k = 0; k < 8; ++k) {
                        const float kc = (float)k - 3.5f;
                        const int pp = 8 * (row0 + row) + k;  // the pixel = phase-1 lane
                        const float2 ga = x[pp * TB_ROW + ci];  // (G, alpha * T)
                        const float4 gp = Wp.g[pp];
                        m0 += ga.x;
                        m1 = fmaf(kc, ga.x, m1);
                        m2 = fmaf(kc * kc, ga.x, m2);
                        acc[5] = fmaf(ga.y, gp.x, acc[5]);
                        acc[6] = fmaf(ga.y, gp.y, acc[6]);
                        acc[7] = fmaf(ga.y, gp.z, acc[7]);
                        if (DEPTH) acc[11] = fmaf(ga.y, gp.w, acc[11]);  // sum alpha T gd: dL/dz of the splat
                        if (STATS) {
                            const float vs0 = ga.x * fmaf(ca, kc, q0r), vs1 = ga.x * fmaf(cb, kc, q1r);
                            const float mm = vs0 * vs0 + vs1 * vs1;
                            acc[9] += EXACT_EXP ? sqrtf(mm) : sqrt_approx(mm);
                            acc[10] += ga.y > 0.0f ? 1.0f : 0.0f;  // alpha >= 1/255 and T > 0: alpha*T > 0 exactly for the contributing pixels
                        }
                        nz |= __float_as_uint(ga.y);
                    }
                    // t = sum G q, u = sum kc G q; sum G q0 q0 = q0r t0 + a u0, sum G q0 q1 = q1r t0 + b u0, sum G q1 q1 = q1r t1 + b u1
                    const float t0 = fmaf(ca, m1, q0r * m0), t1 = fmaf(cb, m1, q1r * m0);
                    const float u0 = fmaf(ca, m2, q0r * m1), u1 = fmaf(cb, m2, q1r * m1);
                    acc[0] += t0;
                    acc[1] += t1;
                    acc[2] += fmaf(ca, u0, q0r * t0);  // the 1/2 of UT:345 is applied once per point in the epilogue kernel
                    acc[3] += fmaf(cb, u0, q1r * t0);
                    acc[4] += fmaf(cb, u1, q1r * t1);
                    acc[8] += m0;
                }
                if constexpr (CF > 0) {  // a loop of its own (alpha T re-read): the CF sums would not fit beside the moments' registers
#pragma unroll 1
                    for (int row = 0; row < TB_ROWS; ++row) {
#pragma unroll 4
                        for (int k = 0; k < 8; ++k) {
                            const int pp = 8 * (row0 + row) + k;
                            const float aT = x[pp * TB_ROW + ci].y;
#pragma unroll
                            for (int c = 0; c < CF; c += 4) {
                                const float4 gc = WF.g[pp][c / 4];
                                af[c] = fmaf(aT, gc.x, af[c]);
                                af[c + 1] = fmaf(aT, gc.y, af[c + 1]);
                                af[c + 2] = fmaf(aT, gc.z, af[c + 2]);
                                af[c + 3] = fmaf(aT, gc.w, af[c + 3]);
                            }
                        }
                    }
                }
                // the lanes of the splat: rows 0..3 of the patch
#pragma unroll
                for (int d = TB_CHUNK; d < 32; d *= 2) {
#pragma unroll
                    for (int k = 0; k < NV; ++k) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], d);
                    if (DEPTH) acc[11] += __shfl_xor_sync(0xffffffffu, acc[11], d);
                    if constexpr (CF > 0) {
#pragma unroll
                        for (int c = 0; c < CF; ++c) af[c] += __shfl_xor_sync(0xffffffffu, af[c], d);
                    }
                    nz |= __shfl_xor_sync(0xffffffffu, nz, d);
                }
                if constexpr (CF > 0) if (active && nz != 0u) {
                    // the 32 / TB_CHUNK lanes of the splat hold the same sums: lane part h adds the float4 groups q with
                    // q % parts == h (one 16-byte RED per group when the rows are 16-byte aligned, C % 4 == 0)
                    constexpr int parts = 32 / TB_CHUNK;
                    const int h = lane / TB_CHUNK;
                    float *dst = fp.grad_features + (size_t)WF.row[ci] * C;
#pragma unroll
                    for (int c = 0; c < CF; c += 4) {
                        if ((c / 4) % parts != h || c >= C) continue;
                        if (C % 4 == 0) {
                            red_add_f32x4(dst + c, make_float4(af[c], af[c + 1], af[c + 2], af[c + 3]));
                        } else {
#pragma unroll
                            for (int k = 0; k < 4; ++k)
                                if (c + k < C) atomicAdd(dst + c + k, af[c + k]);
                        }
                    }
                }
                acc[8] *= EXACT_EXP ? (1.0f - s1.z) : s1.z;  // d alpha / d logit = alpha (1 - opacity)
                __syncwarp();  // every lane has consumed its exchange entries: the buffer now takes the finished rows
                if (lane < TB_CHUNK) {
                    if (!(active && nz != 0u)) ck_off[ci] = -1;
                    else GSB_EMU_COUNT(EC_TB_ROWS, 1);
                    // the whole 12-word row (words NV..10 are zero, and 11 without DEPTH): 48 B apart, so the 8 lanes of a
                    // quarter-warp cover the 32 banks once per float4
                    fin[3 * ci] = make_float4(acc[0], acc[1], acc[2], acc[3]);
                    fin[3 * ci + 1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
                    fin[3 * ci + 2] = make_float4(acc[8], STATS ? acc[9] : 0.0f, STATS ? acc[10] : 0.0f,
                                                  DEPTH ? acc[11] : 0.0f);
                }
                __syncwarp();
                // float4 e of the chunk's finished rows goes to word 4 (e % 3) of row e / 3: the same 2 sectors per row
                // as 12 scalar REDs, in 3 vector REDs
#pragma unroll
                for (int e0 = 0; e0 < 3 * TB_CHUNK; e0 += 32) {
                    const int e = e0 + lane, row = e / 3;
                    if (e < 3 * TB_CHUNK) {
                        const int o = ck_off[row];
                        if (o >= 0) red_add_f32x4(p.accum + (size_t)o * GSB_ACCUM_FLOATS + 4 * (e - 3 * row), fin[e]);
                    }
                }
                __syncwarp();  // the next chunk overwrites the chunk buffer and the exchange buffer
            }
        } while (pos < count);
        if (!real) break;
    }
    if (STATS) {
        p.mag_image[2 * pix] = mag0;  // GPCR:700-704
        p.mag_image[2 * pix + 1] = mag1;
    }
    if (COUNT) {
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            n_visits += __shfl_xor_sync(0xffffffffu, n_visits, d);
            n_pairs += __shfl_xor_sync(0xffffffffu, n_pairs, d);
        }
        if (lane == 0) {
            atomicAdd(p.work_counters, (unsigned long long)n_visits);
            atomicAdd(p.work_counters + 1, (unsigned long long)n_pairs);
        }
    }
}

#ifndef GSB_HOST_EMU
template <bool EXACT_EXP, bool STATS, bool DEPTH = false, bool ALPHA = false, int CF = 0, bool WRAP = false>
static int launch_tb(const TbParams<CF> &p, int tiles, cudaStream_t stream) {
    static bool configured = false;  // one device per process (one process per GPU)
    if (!configured) {
        GSB_CUDA_CHECK(cudaFuncSetAttribute(blend_backward_transposed_kernel<EXACT_EXP, STATS, false, DEPTH, ALPHA, CF, WRAP>,
                                            cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tb_smem_bytes<CF>()));
        configured = true;
    }
    blend_backward_transposed_kernel<EXACT_EXP, STATS, false, DEPTH, ALPHA, CF, WRAP>
        <<<tiles, GSB_TILE_PIXELS, tb_smem_bytes<CF>(), stream>>>(p);
    GSB_CUDA_CHECK(cudaGetLastError());
    return GSB_OK;
}

template <bool DEPTH, bool ALPHA, int CF = 0, bool WRAP = false>
static int launch_tb_terms(const TbParams<CF> &p, int tiles, bool exact_exp, bool stats, cudaStream_t stream) {
    if (exact_exp)
        return stats ? launch_tb<true, true, DEPTH, ALPHA, CF, WRAP>(p, tiles, stream)
                     : launch_tb<true, false, DEPTH, ALPHA, CF, WRAP>(p, tiles, stream);
    return stats ? launch_tb<false, true, DEPTH, ALPHA, CF, WRAP>(p, tiles, stream)
                 : launch_tb<false, false, DEPTH, ALPHA, CF, WRAP>(p, tiles, stream);
}

template <int CF, bool WRAP = false>
static int launch_tb_features(const BlendBwdFeatParams &p, int tiles, bool exact_exp, bool stats, cudaStream_t stream, bool depth,
                              bool alpha) {
    if (alpha)
        return depth ? launch_tb_terms<true, true, CF, WRAP>(p, tiles, exact_exp, stats, stream)
                     : launch_tb_terms<false, true, CF, WRAP>(p, tiles, exact_exp, stats, stream);
    return depth ? launch_tb_terms<true, false, CF, WRAP>(p, tiles, exact_exp, stats, stream)
                 : launch_tb_terms<false, false, CF, WRAP>(p, tiles, exact_exp, stats, stream);
}

template <bool WRAP>
static int launch_tb_all(const BlendBwdParams &p, int tiles, bool exact_exp, bool stats, cudaStream_t stream, bool depth,
                         bool alpha, const BlendFeatureParams *feat) {
    if (feat) {
        BlendBwdFeatParams fp;
        static_cast<BlendBwdParams &>(fp) = p;
        fp.feat = *feat;
        const int C = feat->channels;
        return C <= 4 ? launch_tb_features<4, WRAP>(fp, tiles, exact_exp, stats, stream, depth, alpha)
             : C <= 8 ? launch_tb_features<8, WRAP>(fp, tiles, exact_exp, stats, stream, depth, alpha)
                      : launch_tb_features<16, WRAP>(fp, tiles, exact_exp, stats, stream, depth, alpha);
    }
    if (alpha)
        return depth ? launch_tb_terms<true, true, 0, WRAP>(p, tiles, exact_exp, stats, stream)
                     : launch_tb_terms<false, true, 0, WRAP>(p, tiles, exact_exp, stats, stream);
    return depth ? launch_tb_terms<true, false, 0, WRAP>(p, tiles, exact_exp, stats, stream)
                 : launch_tb_terms<false, false, 0, WRAP>(p, tiles, exact_exp, stats, stream);
}

// depth = true: p.grad_depth and p.depth must be set (the DEPTH instantiations); alpha = true: p.grad_alpha (ALPHA);
// feat: the feature channels, C in 1..16 (the CF instantiation of width 4, 8 or 16), or NULL; wrap: the WRAP instantiations
// (an equirectangular frame)
int launch_blend_backward_transposed(const BlendBwdParams &p, int tiles, bool exact_exp, bool stats,
                                     cudaStream_t stream, bool depth, bool alpha, const BlendFeatureParams *feat, bool wrap) {
    return wrap ? launch_tb_all<true>(p, tiles, exact_exp, stats, stream, depth, alpha, feat)
                : launch_tb_all<false>(p, tiles, exact_exp, stats, stream, depth, alpha, feat);
}

// Diagnostic: loop A with GPU-side work counters (default arithmetic, no hook statistics): counters[0] = (warp, splat)
// visits of phase 1, [1] = contributing (pixel, splat) pairs.  Adds into p.accum like the normal launch.
int launch_blend_backward_count(const BlendBwdParams &p, int tiles, cudaStream_t stream) {
    GSB_CUDA_CHECK(cudaFuncSetAttribute(blend_backward_transposed_kernel<false, false, true>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TbShared)));
    blend_backward_transposed_kernel<false, false, true><<<tiles, GSB_TILE_PIXELS, sizeof(TbShared), stream>>>(p);
    GSB_CUDA_CHECK(cudaGetLastError());
    return GSB_OK;
}
#endif  // GSB_HOST_EMU

}  // namespace gsb
