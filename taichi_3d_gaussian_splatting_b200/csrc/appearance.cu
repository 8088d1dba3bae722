// appearance.cu -- per-view appearance compensation: slicing a bilateral grid (Wang et al., "Bilateral Guided Radiance
// Field Processing", SIGGRAPH 2024), its gradient and its total-variation prior.  For one view, G is (12, Gz, Gy, Gx), a
// 3x4 affine [A | b] (row-major) per node over (x, y, luminance).  At pixel (px, py) of an (H,W,3) image with colour c:
//   gx = px (Gx-1) / max(W-1, 1),  gy = py (Gy-1) / max(H-1, 1),  gz = clamp(0.299 c_r + 0.587 c_g + 0.114 c_b, 0, 1) (Gz-1)
//   [A | b] = trilinear interpolation of G at (gx, gy, gz), the lower corner index clamped to n-2;  out = A c + b
// (= F.grid_sample(G[None], (x, y, 2 lum - 1), align_corners=True, padding_mode="border")).
//
// The work is split by grid CELL: the pixels whose lower (x, y) corner is (cx, cy) form a rectangle of the image, and they
// read only the cell's 4 (x, y) nodes.  One CTA handles a chunk of BG_CHUNK pixels of one cell (the cells x chunks grid is
// fixed by the shapes), with those 4 x Gz x 12 node values staged in shared memory.
//   forward:   pixel-parallel inside the cell.
//   backward:  dL/dc (in place over dL/dout: each pixel's gradient is read and written by the same thread) and the cell's
//              dL/dG.  Each warp keeps a private (Gz, 4 corners x 12) histogram in shared memory: the warp's 32 pixels are
//              staged, then visited in lane order, each lane owning one or two (corner, channel) columns -- no atomics.  The
//              CTA adds its 8 warp histograms in warp order into its row of partials; bilateral_grid_finish_kernel adds a
//              node's partials (its <= 4 cells, each with its chunks) with one warp in a fixed order.  Two calls are
//              bit-identical.
//   TV:        tv(G) = sum over the x, y and z axes of mean((G[i+1] - G[i])^2); one CTA adds w dtv/dG into dL/dG and writes
//              w tv in a fixed summation order.
#include <initializer_list>

#include "common.cuh"

namespace gsb {

constexpr int BG_THREADS = 256;
constexpr int BG_WARPS = BG_THREADS / 32;
constexpr int BG_CHUNK = BG_THREADS * 8;  // pixels of one cell per CTA
constexpr int BG_PIX = 19;                // staged floats per pixel: dcoef[12], corner weights[4], z0, fz (+1 pad: odd stride)
constexpr int TV_THREADS = 256;

struct BilateralGridParams {
    const float *image;     // (H,W,3) slice input
    const float *grid;      // (12,Gz,Gy,Gx)
    float *out;             // (H,W,3) forward output
    const float *grad_out;  // (H,W,3) dL/dout (backward)
    float *grad_in;         // (H,W,3) dL/dimage, may alias grad_out
    float *partials;        // [blocks][4 corners][Gz][12] (backward)
    float *grad_grid;       // (12,Gz,Gy,Gx) (finish, TV)
    float *tv_out;          // device float: w tv (TV)
    float tv_weight;
    int H, W, gx, gy, gz;
    int ncx, ncy, chunks;   // cells along x and y, CTAs per cell
};

// the node coordinate of pixel p along an axis of L pixels and n nodes, its lower corner (clamped to n-2) and fraction
__host__ __device__ __forceinline__ float bg_coord(int p, int n, int L) {
    return (float)(p * (n - 1)) / (float)(L > 1 ? L - 1 : 1);
}
__host__ __device__ __forceinline__ int bg_lower(float g, int n) {
    const int hi = n > 2 ? n - 2 : 0;
    int i = (int)floorf(g);
    return i < 0 ? 0 : (i > hi ? hi : i);
}
// the first pixel whose lower corner is >= c (c in 0..cells; cells = max(n-1, 1))
__host__ __device__ __forceinline__ int bg_cell_start(int c, int n, int L) {
    if (c <= 0) return 0;
    if (c >= (n > 1 ? n - 1 : 1)) return L;
    int p = (int)(((long long)c * (L - 1)) / (n - 1));
    while (p > 0 && bg_lower(bg_coord(p - 1, n, L), n) >= c) --p;
    while (p < L && bg_lower(bg_coord(p, n, L), n) < c) ++p;
    return p;
}

// the 12 coefficients at one pixel from the staged cell nodes s[corner][z][12], and (slope != null) their derivative in gz
__device__ __forceinline__ void bg_coefficients(const float *s, int gz, float fx, float fy, int z0, int z1, float fz,
                                                float coef[12], float *slope) {
    const float w[4] = {(1.0f - fx) * (1.0f - fy), fx * (1.0f - fy), (1.0f - fx) * fy, fx * fy};
#pragma unroll
    for (int k = 0; k < 12; ++k) {
        coef[k] = 0.0f;
        if (slope) slope[k] = 0.0f;
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const float *a = s + (c * gz + z0) * 12, *b = s + (c * gz + z1) * 12;
#pragma unroll
        for (int k = 0; k < 12; ++k) {
            const float d = b[k] - a[k];
            coef[k] += w[c] * (a[k] + fz * d);
            if (slope) slope[k] += w[c] * d;
        }
    }
}

__device__ __forceinline__ float bg_luminance(float r, float g, float b) { return 0.299f * r + 0.587f * g + 0.114f * b; }

// the cell of this CTA: its pixel rectangle and its staged nodes; returns the number of pixels of the cell
__device__ __forceinline__ int bg_stage_cell(const BilateralGridParams &p, float *s_node, int *x_lo, int *y_lo, int *w) {
    const int cell = blockIdx.x / p.chunks;
    const int cx = cell % p.ncx, cy = cell / p.ncx;
    *x_lo = bg_cell_start(cx, p.gx, p.W);
    *y_lo = bg_cell_start(cy, p.gy, p.H);
    *w = bg_cell_start(cx + 1, p.gx, p.W) - *x_lo;
    const int h = bg_cell_start(cy + 1, p.gy, p.H) - *y_lo;
    const int x1 = min(cx + 1, p.gx - 1), y1 = min(cy + 1, p.gy - 1);
    const int n = 4 * p.gz * 12;
    for (int i = threadIdx.x; i < n; i += BG_THREADS) {
        const int c = i / (p.gz * 12), z = (i / 12) % p.gz, k = i % 12;
        s_node[i] = __ldg(&p.grid[(((long long)k * p.gz + z) * p.gy + ((c & 2) ? y1 : cy)) * p.gx + ((c & 1) ? x1 : cx)]);
    }
    __syncthreads();
    return *w * h;
}

__device__ __forceinline__ void bg_z(float lum, int gz, int *z0, int *z1, float *fz) {
    const float g = fminf(fmaxf(lum, 0.0f), 1.0f) * (float)(gz - 1);
    *z0 = bg_lower(g, gz);
    *z1 = min(*z0 + 1, gz - 1);
    *fz = g - (float)*z0;
}

__global__ void __launch_bounds__(BG_THREADS) bilateral_grid_forward_kernel(const BilateralGridParams p) {
    __shared__ float s_node[4 * GSB_BILATERAL_GRID_MAX_Z * 12];
    int x_lo, y_lo, w;
    const int n = bg_stage_cell(p, s_node, &x_lo, &y_lo, &w);
    const int begin = (blockIdx.x % p.chunks) * BG_CHUNK, end = min(n, begin + BG_CHUNK);
    for (int i = begin + threadIdx.x; i < end; i += BG_THREADS) {
        const int px = x_lo + i % w, py = y_lo + i / w;
        const long long o = 3 * ((long long)py * p.W + px);
        const float r = __ldg(&p.image[o]), g = __ldg(&p.image[o + 1]), b = __ldg(&p.image[o + 2]);
        const float fx = bg_coord(px, p.gx, p.W) - (float)bg_lower(bg_coord(px, p.gx, p.W), p.gx);
        const float fy = bg_coord(py, p.gy, p.H) - (float)bg_lower(bg_coord(py, p.gy, p.H), p.gy);
        int z0, z1;
        float fz;
        bg_z(bg_luminance(r, g, b), p.gz, &z0, &z1, &fz);
        float coef[12];
        bg_coefficients(s_node, p.gz, fx, fy, z0, z1, fz, coef, nullptr);
        p.out[o] = coef[0] * r + coef[1] * g + coef[2] * b + coef[3];
        p.out[o + 1] = coef[4] * r + coef[5] * g + coef[6] * b + coef[7];
        p.out[o + 2] = coef[8] * r + coef[9] * g + coef[10] * b + coef[11];
    }
}

__global__ void __launch_bounds__(BG_THREADS) bilateral_grid_backward_kernel(const BilateralGridParams p) {
    __shared__ float s_node[4 * GSB_BILATERAL_GRID_MAX_Z * 12];
    __shared__ float s_hist[BG_WARPS][GSB_BILATERAL_GRID_MAX_Z * 48];  // per warp: [z][corner * 12 + channel]
    __shared__ float s_pix[BG_WARPS][32 * BG_PIX];
    int x_lo, y_lo, w;
    const int n = bg_stage_cell(p, s_node, &x_lo, &y_lo, &w);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float *hist = s_hist[warp], *pix = s_pix[warp];
    for (int i = lane; i < p.gz * 48; i += 32) hist[i] = 0.0f;
    // the (corner, channel) columns of this lane: lane and lane + 32 (lanes 0..15)
    const int col0 = lane, col1 = lane + 32;
    const int c0 = col0 / 12, k0 = col0 % 12, c1 = col1 / 12, k1 = col1 % 12;
    const int begin = (blockIdx.x % p.chunks) * BG_CHUNK + warp * (BG_CHUNK / BG_WARPS);
    const int end = min(n, begin + BG_CHUNK / BG_WARPS);
    for (int base = begin; base < end; base += 32) {
        const int i = base + lane;
        float *mine = pix + lane * BG_PIX;
        if (i < end) {
            const int px = x_lo + i % w, py = y_lo + i / w;
            const long long o = 3 * ((long long)py * p.W + px);
            const float r = __ldg(&p.image[o]), g = __ldg(&p.image[o + 1]), b = __ldg(&p.image[o + 2]);
            const float g0 = p.grad_out[o], g1 = p.grad_out[o + 1], g2 = p.grad_out[o + 2];
            const float fx = bg_coord(px, p.gx, p.W) - (float)bg_lower(bg_coord(px, p.gx, p.W), p.gx);
            const float fy = bg_coord(py, p.gy, p.H) - (float)bg_lower(bg_coord(py, p.gy, p.H), p.gy);
            const float lum = bg_luminance(r, g, b);
            int z0, z1;
            float fz;
            bg_z(lum, p.gz, &z0, &z1, &fz);
            float coef[12], slope[12];
            bg_coefficients(s_node, p.gz, fx, fy, z0, z1, fz, coef, slope);
            const float gi[3] = {g0, g1, g2}, cj[4] = {r, g, b, 1.0f};
            float dz = 0.0f;
#pragma unroll
            for (int a = 0; a < 3; ++a) {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float d = gi[a] * cj[j];
                    mine[4 * a + j] = d;
                    dz += d * slope[4 * a + j];
                }
            }
            // through the clamp of the luminance: zero where it is active
            const float dlum = (lum > 0.0f && lum < 1.0f) ? dz * (float)(p.gz - 1) : 0.0f;
            p.grad_in[o] = coef[0] * g0 + coef[4] * g1 + coef[8] * g2 + dlum * 0.299f;
            p.grad_in[o + 1] = coef[1] * g0 + coef[5] * g1 + coef[9] * g2 + dlum * 0.587f;
            p.grad_in[o + 2] = coef[2] * g0 + coef[6] * g1 + coef[10] * g2 + dlum * 0.114f;
            mine[12] = (1.0f - fx) * (1.0f - fy);
            mine[13] = fx * (1.0f - fy);
            mine[14] = (1.0f - fx) * fy;
            mine[15] = fx * fy;
            mine[16] = (float)z0;
            mine[17] = fz;
        }
        __syncwarp();
        const int count = min(32, end - base);
        for (int j = 0; j < count; ++j) {
            const float *q = pix + j * BG_PIX;
            const int z0 = (int)q[16];
            const float fz = q[17];
            {
                const float v = q[12 + c0] * q[k0];
                hist[z0 * 48 + col0] += v * (1.0f - fz);
                if (p.gz > 1) hist[(z0 + 1) * 48 + col0] += v * fz;
            }
            if (col1 < 48) {
                const float v = q[12 + c1] * q[k1];
                hist[z0 * 48 + col1] += v * (1.0f - fz);
                if (p.gz > 1) hist[(z0 + 1) * 48 + col1] += v * fz;
            }
        }
        __syncwarp();
    }
    __syncthreads();
    // this CTA's row of partials, [corner][z][channel]: the warp histograms added in warp order
    float *row = p.partials + (long long)blockIdx.x * 4 * p.gz * 12;
    for (int e = threadIdx.x; e < 4 * p.gz * 12; e += BG_THREADS) {
        const int c = e / (p.gz * 12), z = (e / 12) % p.gz, k = e % 12;
        float s = 0.0f;
#pragma unroll
        for (int v = 0; v < BG_WARPS; ++v) s += s_hist[v][z * 48 + c * 12 + k];
        row[e] = s;
    }
}

// dL/dG[k, z, y, x], one warp per node value: the node's partials -- its cells (cy, then cx, then the corner), each with
// its chunks -- listed in that fixed order; lane l adds items l, l + 32, ... in order, then a fixed butterfly adds the lanes
__global__ void __launch_bounds__(BG_THREADS) bilateral_grid_finish_kernel(const BilateralGridParams p) {
    const int n = 12 * p.gz * p.gy * p.gx;
    const int lane = threadIdx.x & 31;
    for (int e = (blockIdx.x * BG_THREADS + threadIdx.x) >> 5; e < n; e += (gridDim.x * BG_THREADS) >> 5) {
        const int x = e % p.gx, y = (e / p.gx) % p.gy, z = (e / (p.gx * p.gy)) % p.gz, k = e / (p.gx * p.gy * p.gz);
        float s = 0.0f;
        int item = 0;
        for (int cy = max(y - 1, 0); cy <= min(y, p.ncy - 1); ++cy) {
            for (int by = 0; by < 2; ++by) {
                if ((by ? min(cy + 1, p.gy - 1) : cy) != y) continue;
                for (int cx = max(x - 1, 0); cx <= min(x, p.ncx - 1); ++cx) {
                    for (int bx = 0; bx < 2; ++bx) {
                        if ((bx ? min(cx + 1, p.gx - 1) : cx) != x) continue;
                        const float *src = p.partials + (long long)(cy * p.ncx + cx) * p.chunks * 4 * p.gz * 12 +
                                           ((bx | (by << 1)) * p.gz + z) * 12 + k;
                        // this cell's chunks are items item .. item + chunks - 1 of the node's list
                        for (int ch = ((lane - item) % 32 + 32) % 32; ch < p.chunks; ch += 32)
                            s += src[(long long)ch * 4 * p.gz * 12];
                        item += p.chunks;
                    }
                }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) p.grad_grid[e] = s;
    }
}

// one CTA: grad_grid += w dtv/dG, tv_out = w tv (per-thread double sums, then the warp sums in order)
__global__ void __launch_bounds__(TV_THREADS) bilateral_grid_tv_kernel(const BilateralGridParams p) {
    __shared__ double s_part[TV_THREADS / 32];
    const int n = 12 * p.gz * p.gy * p.gx;
    const int dims[3] = {p.gx, p.gy, p.gz}, strides[3] = {1, p.gx, p.gx * p.gy};
    float scale[3];  // 2 w / (number of differences along the axis)
    double inv[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const long long m = dims[a] > 1 ? (long long)n / dims[a] * (dims[a] - 1) : 0;
        inv[a] = m ? 1.0 / (double)m : 0.0;
        scale[a] = m ? (float)(2.0 * (double)p.tv_weight / (double)m) : 0.0f;
    }
    double acc = 0.0;
    for (int e = threadIdx.x; e < n; e += TV_THREADS) {
        const float v = p.grid[e];
        float g = 0.0f;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            if (dims[a] < 2) continue;
            const int i = (e / strides[a]) % dims[a];
            if (i > 0) g += scale[a] * (v - p.grid[e - strides[a]]);
            if (i + 1 < dims[a]) {
                const float d = p.grid[e + strides[a]] - v;
                g -= scale[a] * d;
                acc += (double)(d * d) * inv[a];
            }
        }
        p.grad_grid[e] += g;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int v = 0; v < TV_THREADS / 32; ++v) t += s_part[v];
        *p.tv_out = (float)((double)p.tv_weight * t);
    }
}

// the launch shape of one (H, W, Gx, Gy, Gz): cells along x and y, and CTAs per cell (the largest cell's pixels / BG_CHUNK)
static inline void bilateral_grid_shape(int H, int W, int gx, int gy, int gz, BilateralGridParams *p) {
    p->H = H;
    p->W = W;
    p->gx = gx;
    p->gy = gy;
    p->gz = gz;
    p->ncx = gx > 1 ? gx - 1 : 1;
    p->ncy = gy > 1 ? gy - 1 : 1;
    int mw = 0, mh = 0;
    for (int c = 0; c < p->ncx; ++c) mw = max(mw, bg_cell_start(c + 1, gx, W) - bg_cell_start(c, gx, W));
    for (int c = 0; c < p->ncy; ++c) mh = max(mh, bg_cell_start(c + 1, gy, H) - bg_cell_start(c, gy, H));
    const long long most = (long long)mw * mh;
    p->chunks = (int)max(1LL, (most + BG_CHUNK - 1) / BG_CHUNK);
}

static inline int bilateral_grid_blocks(const BilateralGridParams &p) { return p.ncx * p.ncy * p.chunks; }

static inline bool bilateral_grid_shape_ok(int H, int W, int gx, int gy, int gz) {
    return H >= 1 && W >= 1 && gx >= 1 && gx <= GSB_BILATERAL_GRID_MAX_XY && gy >= 1 && gy <= GSB_BILATERAL_GRID_MAX_XY &&
           gz >= 1 && gz <= GSB_BILATERAL_GRID_MAX_Z;
}

static inline long long bilateral_grid_temp_bytes(int H, int W, int gx, int gy, int gz) {
    if (!bilateral_grid_shape_ok(H, W, gx, gy, gz)) return 0;
    BilateralGridParams p;
    bilateral_grid_shape(H, W, gx, gy, gz, &p);
    return ((long long)bilateral_grid_blocks(p) * 4 * gz * 12 * 4 + 255) / 256 * 256;
}

#ifndef GSB_HOST_EMU
static inline int bilateral_grid_finish_blocks(int gx, int gy, int gz) {  // one warp per node value, at most 8 per SM
    const long long b = (12LL * gx * gy * gz + BG_WARPS - 1) / BG_WARPS, cap = 8LL * num_sms();
    return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

int launch_bilateral_grid_forward(const float *image, const float *grid, int H, int W, int gx, int gy, int gz, float *out,
                                  cudaStream_t stream) {
    BilateralGridParams p = {};
    bilateral_grid_shape(H, W, gx, gy, gz, &p);
    p.image = image;
    p.grid = grid;
    p.out = out;
    bilateral_grid_forward_kernel<<<bilateral_grid_blocks(p), BG_THREADS, 0, stream>>>(p);
    GSB_CUDA_CHECK(cudaGetLastError());
    return GSB_OK;
}

int launch_bilateral_grid_backward(const float *image, const float *grid, int H, int W, int gx, int gy, int gz,
                                   const float *grad_out, float *grad_in, float *grad_grid, void *temp, float tv_weight,
                                   float *tv_out, cudaStream_t stream) {
    BilateralGridParams p = {};
    bilateral_grid_shape(H, W, gx, gy, gz, &p);
    p.image = image;
    p.grid = grid;
    p.grad_out = grad_out;
    p.grad_in = grad_in;
    p.partials = static_cast<float *>(temp);
    p.grad_grid = grad_grid;
    p.tv_out = tv_out;
    p.tv_weight = tv_weight;
    bilateral_grid_backward_kernel<<<bilateral_grid_blocks(p), BG_THREADS, 0, stream>>>(p);
    GSB_CUDA_CHECK(cudaGetLastError());
    bilateral_grid_finish_kernel<<<bilateral_grid_finish_blocks(gx, gy, gz), BG_THREADS, 0, stream>>>(p);
    GSB_CUDA_CHECK(cudaGetLastError());
    if (tv_out) {
        bilateral_grid_tv_kernel<<<1, TV_THREADS, 0, stream>>>(p);
        GSB_CUDA_CHECK(cudaGetLastError());
    }
    return GSB_OK;
}
#endif

}  // namespace gsb

#ifndef GSB_HOST_EMU
extern "C" {

int64_t gsb200_bilateral_grid_temp_bytes(int32_t camera_height, int32_t camera_width, int32_t grid_x, int32_t grid_y,
                                         int32_t grid_z) {
    return gsb::bilateral_grid_temp_bytes(camera_height, camera_width, grid_x, grid_y, grid_z);
}

static int bilateral_grid_check(const char *what, int H, int W, int gx, int gy, int gz,
                                std::initializer_list<const void *> pointers) {
    if (!gsb::bilateral_grid_shape_ok(H, W, gx, gy, gz)) {
        gsb::set_error("%s: H, W >= 1, 1 <= Gx, Gy <= %d and 1 <= Gz <= %d (got H=%d W=%d grid %dx%dx%d)", what,
                       GSB_BILATERAL_GRID_MAX_XY, GSB_BILATERAL_GRID_MAX_Z, H, W, gx, gy, gz);
        return GSB_EINVAL;
    }
    for (const void *q : pointers) {
        if (!q || reinterpret_cast<uintptr_t>(q) % 4) {
            gsb::set_error("%s: null or misaligned pointer", what);
            return GSB_EINVAL;
        }
    }
    return GSB_OK;
}

int gsb200_bilateral_grid_forward(const float *image, const float *grid, int32_t camera_height, int32_t camera_width,
                                  int32_t grid_x, int32_t grid_y, int32_t grid_z, float *image_out, void *stream) {
    const int rc = bilateral_grid_check("bilateral_grid_forward", camera_height, camera_width, grid_x, grid_y, grid_z,
                                        {image, grid, image_out});
    if (rc != GSB_OK) return rc;
    return gsb::launch_bilateral_grid_forward(image, grid, camera_height, camera_width, grid_x, grid_y, grid_z, image_out,
                                              static_cast<cudaStream_t>(stream));
}

int gsb200_bilateral_grid_backward(const float *image, const float *grid, int32_t camera_height, int32_t camera_width,
                                   int32_t grid_x, int32_t grid_y, int32_t grid_z, const float *grad_image_out,
                                   float *grad_image, float *grad_grid, void *temp, int64_t temp_bytes, void *stream) {
    int rc = bilateral_grid_check("bilateral_grid_backward", camera_height, camera_width, grid_x, grid_y, grid_z,
                                  {image, grid, grad_image_out, grad_image, grad_grid});
    if (rc != GSB_OK) return rc;
    if (!temp || reinterpret_cast<uintptr_t>(temp) % 16 ||
        temp_bytes < gsb::bilateral_grid_temp_bytes(camera_height, camera_width, grid_x, grid_y, grid_z)) {
        gsb::set_error("bilateral_grid_backward: temp null, not 16-byte aligned or smaller than "
                       "gsb200_bilateral_grid_temp_bytes (temp_bytes=%lld)", (long long)temp_bytes);
        return GSB_EINVAL;
    }
    return gsb::launch_bilateral_grid_backward(image, grid, camera_height, camera_width, grid_x, grid_y, grid_z,
                                               grad_image_out, grad_image, grad_grid, temp, 0.0f, nullptr,
                                               static_cast<cudaStream_t>(stream));
}

}  // extern "C"
#endif  // GSB_HOST_EMU
