// sort.cu -- device LSD radix sort of (tile | depth) keys with the in-camera offset as payload
// (replaces torch.sort + gather, GPCR:947-950) and the per-tile range detection (GPCR:175-193).
//
// One-sweep organisation: one histogram kernel builds the digit histograms of every pass (and their exclusive
// prefixes); each pass is a single kernel in which a CTA (a) pulls its 3072-key tile into shared memory with one
// TMA bulk copy (cp.async.bulk + mbarrier -> SASS UBLKCP), (b) ranks the keys stably with
// per-bit warp ballots, (c) obtains the global digit offsets by a per-digit decoupled look-back
// over the preceding CTAs, and (d) scatters keys and payloads from a block-sorted shared-memory
// staging area so that global stores go out in runs.  Keys are only as wide as the live bits:
// ceil(log2 T) tile bits + the bits of int(far*scale); 32-bit keys whenever that is <= 32 bits.
// Stability (ties keep ascending in-camera offset = ascending point id) is what reproduces the
// reference's blend order.  HBM-bound: 2*(key+4) B per key per pass + one key read for histograms.
#include "common.cuh"

namespace gsb {

constexpr unsigned int SS_AGGREGATE = 1u << 30;
constexpr unsigned int SS_INCLUSIVE = 2u << 30;
constexpr unsigned int SS_VALUE_MASK = (1u << 30) - 1;
#ifndef GSB_SORT_LOOKBACK
#define GSB_SORT_LOOKBACK 4
#endif
constexpr int LOOKBACK = GSB_SORT_LOOKBACK;  // predecessors whose state is fetched per look-back round
constexpr int RBITS = 8;                     // digit width
constexpr int RADIX = 1 << RBITS;            // = SORT_BLOCK_THREADS: thread t owns digit t
static_assert(RADIX == SORT_BLOCK_THREADS, "one digit per thread");

// Digit width for a key of `bits` live bits.  10-bit digits would save a pass at C3 but need 1024-bin ranking and 4 KB
// of look-back state per CTA, so 8 bits are always used.
int sort_radix_bits(int bits) {
    (void)bits;
    return RBITS;
}

__device__ __forceinline__ unsigned int ld_u32_volatile(const unsigned int *p) {
    return *reinterpret_cast<const volatile unsigned int *>(p);
}
__device__ __forceinline__ void st_u32_volatile(unsigned int *p, unsigned int v) {
    *reinterpret_cast<volatile unsigned int *>(p) = v;
}

// The lanes of the warp whose v (< 2^(RBITS+1)) equals this lane's: what __match_any_sync(0xffffffff, v) returns, built from
// one ballot per bit.  MATCH.ANY costs more the more distinct values the warp holds: with it the ranking loop of the later
// passes, whose keys are no longer grouped by splat, took about three times as long as in the first pass.
__device__ __forceinline__ unsigned int match_digit(int v) {
    unsigned int peers = 0xffffffffu;
#pragma unroll
    for (int b = 0; b <= RBITS; ++b) {
        const bool bit = (v >> b) & 1;
        const unsigned int set = __ballot_sync(0xffffffffu, bit);
        peers &= bit ? set : ~set;
    }
    return peers;
}

// ------------------------------------------------------------------ live-bit compaction
// A key is  tile << depth_bits | depth_key.  depth_bits is sized for the FAR PLANE (int(far * scale): 17 bits with the
// reference's defaults), but a frame only uses bit_width(max depth key over its in-camera points) of them -- 10 at
// BASELINE config 3.  The per-point kernel leaves that maximum in the workspace (one atomicMax per CTA), and every sort
// kernel reads it and sorts the COMPACTED key  tile << live_depth_bits | depth_key  instead: its 8-bit digits are cut out
// of the stored key with two shift-and-mask pairs (a digit may straddle the depth / tile boundary).  Same order, same
// stability, ceil((tile_bits + live_depth_bits) / 8) passes instead of ceil((tile_bits + depth_bits) / 8): 3 instead of 4
// at C3.  Which passes run is decided on the device: the host launches the worst-case number, surplus launches exit.
template <typename KeyT>
struct DigitSel {
    int s_lo, s_hi;
    KeyT m_lo, m_hi;
};
template <typename KeyT>
__device__ __forceinline__ int digit_of(KeyT k, const DigitSel<KeyT> &s) {
    return (int)(((k >> s.s_lo) & s.m_lo) | ((k >> s.s_hi) & s.m_hi));
}
__device__ __forceinline__ int live_depth_bits(const int *max_depth_key, int depth_bits) {
    if (!max_depth_key) return depth_bits;
    unsigned int m = (unsigned int)*max_depth_key;
    int b = 0;
    while (m) {
        ++b;
        m >>= 1;
    }
    return b < depth_bits ? b : depth_bits;
}
// number of passes over keys of `end_bit` stored bits whose low `depth_bits` hold `live` live bits
__device__ __forceinline__ int active_passes(int end_bit, int depth_bits, int live) {
    const int total = end_bit - depth_bits + live;
    const int p = (total + RBITS - 1) / RBITS;
    return p < 1 ? 1 : p;
}
template <typename KeyT>
__device__ __forceinline__ DigitSel<KeyT> make_digit_sel(int pass, int depth_bits, int live) {
    // compact bits [lo, lo + 8): those below `live` are stored bits [lo, ...); the others are stored bits
    // depth_bits + (compact bit - live).  Stored bits at or above end_bit are zero, so no upper clamp is needed.
    const int lo = pass * RBITS;
    int n_lo = live - lo;
    n_lo = n_lo < 0 ? 0 : (n_lo > RBITS ? RBITS : n_lo);
    DigitSel<KeyT> s;
    s.s_lo = n_lo > 0 ? lo : 0;
    s.m_lo = (KeyT)((1u << n_lo) - 1u);
    const int first = lo > live ? lo : live;          // first compact bit taken from the tile field
    const int n_hi = RBITS - n_lo;
    s.s_hi = depth_bits + first - live - n_lo;        // >= 0 (see DESIGN section 3)
    s.m_hi = (KeyT)(((1u << n_hi) - 1u) << n_lo);
    if (s.s_hi > (int)sizeof(KeyT) * 8 - 1) {          // digit entirely above the key: contributes nothing
        s.s_hi = 0;
        s.m_hi = 0;
    }
    return s;
}

// ------------------------------------------------------------------ histograms of all passes
// One sweep over the keys builds the digit histograms of every active pass in shared memory; the block that finishes
// last turns each histogram into its exclusive prefix in place, so a pass kernel reads the global base of digit d
// directly (hist[pass * 256 + d]) instead of scanning the 256 bins again in each of its CTAs.
// With `state` set it also zeroes the look-back state the passes will use -- of the active passes only, and of the CTAs that
// have keys -- a few MB per frame where a memset sized for the key capacity would clear every pass of every CTA.
template <typename KeyT>
__global__ void __launch_bounds__(SORT_BLOCK_THREADS)
sort_histogram_kernel(const KeyT *__restrict__ keys, const long long *__restrict__ n_dev, long long capacity,
                      int depth_bits, int end_bit, const int *__restrict__ max_depth_key,
                      unsigned int *__restrict__ hist, unsigned int *__restrict__ done_ctr,
                      unsigned int *__restrict__ state = nullptr, long long state_pass_words = 0) {
    __shared__ unsigned int s_hist[8 * RADIX];
    __shared__ unsigned int s_scan[SORT_BLOCK_THREADS / 32];
    __shared__ unsigned int s_last;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int live = live_depth_bits(max_depth_key, depth_bits);
    const int passes = active_passes(end_bit, depth_bits, live);
    for (int i = tid; i < passes * RADIX; i += SORT_BLOCK_THREADS) s_hist[i] = 0;
    __syncthreads();
    long long n = *n_dev;
    if (n > capacity) n = capacity;
    if (state) {  // [pass][blk][RADIX]: RADIX words (64 uint4) per CTA, state_pass_words per pass
        const long long per_pass = (n + SORT_TILE - 1) / SORT_TILE * (RADIX / 4);
        for (long long k = (long long)blockIdx.x * SORT_BLOCK_THREADS + tid; k < passes * per_pass;
             k += (long long)gridDim.x * SORT_BLOCK_THREADS) {
            const long long p = k / per_pass;
            reinterpret_cast<uint4 *>(state + p * state_pass_words)[k - p * per_pass] = make_uint4(0u, 0u, 0u, 0u);
        }
    }
    DigitSel<KeyT> sel[8];
#pragma unroll
    for (int p = 0; p < 8; ++p) sel[p] = make_digit_sel<KeyT>(p, depth_bits, live);
    // 16 bytes per load and HIST_U loads in flight per thread: with one 4-byte load per trip the sweep is bound by the load
    // latency (8 KB in flight per SM), not by the shared-memory atomics
    constexpr int VEC = 16 / (int)sizeof(KeyT), HIST_U = 2;
    const long long stride = (long long)gridDim.x * SORT_BLOCK_THREADS;
    const long long nvec = n / VEC;  // the key buffers are 16-byte aligned (workspace: 256; gsb200_sort_pairs checks keys_in)
    const uint4 *const kv = reinterpret_cast<const uint4 *>(keys);
    for (long long i = (long long)blockIdx.x * SORT_BLOCK_THREADS + tid; i < nvec; i += HIST_U * stride) {
        uint4 v[HIST_U];
#pragma unroll
        for (int u = 0; u < HIST_U; ++u)
            if (i + u * stride < nvec) v[u] = kv[i + u * stride];
#pragma unroll
        for (int u = 0; u < HIST_U; ++u) {
            if (i + u * stride >= nvec) continue;
            KeyT kk[VEC];
            if (sizeof(KeyT) == 4) {
                kk[0] = (KeyT)v[u].x; kk[1] = (KeyT)v[u].y; kk[VEC - 2] = (KeyT)v[u].z; kk[VEC - 1] = (KeyT)v[u].w;
            } else {
                kk[0] = (KeyT)v[u].x | ((KeyT)v[u].y << (4 * sizeof(KeyT)));
                kk[VEC - 1] = (KeyT)v[u].z | ((KeyT)v[u].w << (4 * sizeof(KeyT)));
            }
#pragma unroll
            for (int e = 0; e < VEC; ++e)
#pragma unroll
                for (int p = 0; p < 8; ++p)
                    if (p < passes) atomicAdd(&s_hist[p * RADIX + digit_of(kk[e], sel[p])], 1u);
        }
    }
    for (long long i = nvec * VEC + (long long)blockIdx.x * SORT_BLOCK_THREADS + tid; i < n; i += stride) {  // < VEC tail keys
        const KeyT k = keys[i];
#pragma unroll
        for (int p = 0; p < 8; ++p)
            if (p < passes) atomicAdd(&s_hist[p * RADIX + digit_of(k, sel[p])], 1u);
    }
    __syncthreads();
    for (int i = tid; i < passes * RADIX; i += SORT_BLOCK_THREADS) {
        const unsigned int c = s_hist[i];
        if (c) atomicAdd(&hist[i], c);
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) s_last = (atomicAdd(done_ctr, 1u) == gridDim.x - 1) ? 1u : 0u;
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    for (int p = 0; p < passes; ++p) {  // thread t owns digit t
        const unsigned int v = ld_u32_volatile(hist + p * RADIX + tid);
        unsigned int incl = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const unsigned int o = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += o;
        }
        __syncthreads();  // s_scan free
        if (lane == 31) s_scan[warp] = incl;
        __syncthreads();
        unsigned int wprefix = 0;
#pragma unroll
        for (int w = 0; w < SORT_BLOCK_THREADS / 32; ++w)
            if (w < warp) wprefix += s_scan[w];
        hist[p * RADIX + tid] = wprefix + incl - v;
    }
}

// ------------------------------------------------------------------ one radix pass
template <typename KeyT>
struct PassSmem {
    alignas(128) KeyT keys[SORT_TILE];  // TMA destination, later the block-sorted key staging area
    int vals[SORT_TILE];                // block-sorted payload staging area
    unsigned short warp_cnt[SORT_BLOCK_THREADS / 32][RADIX];  // per-warp digit counters (<= 512 each)
    unsigned int digit_start[RADIX];    // exclusive start of each digit inside the block-sorted tile
    unsigned int global_base[RADIX];    // destination of local position p with digit d: global_base[d] + p
    unsigned int scan_tmp[SORT_BLOCK_THREADS / 32];
    unsigned long long mbar;
    unsigned int ticket;
};

// Three buffers: `a` holds the input and is never written, the LAST active pass writes `b`, the passes before it
// alternate between `c` and `b` -- so the sorted list is in `b` whatever the number of active passes turns out to be.
template <typename KeyT>
struct PassParams {
    const KeyT *keys_a;
    const int *vals_a;
    KeyT *keys_b;
    int *vals_b;
    KeyT *keys_c;
    int *vals_c;
    const long long *n_dev;
    long long capacity;
    int pass, depth_bits, end_bit, blocks;
    const int *max_depth_key;    // device; NULL: every depth bit is live
    const unsigned int *hist;    // exclusive digit prefixes of every pass: [pass][RADIX]
    unsigned int *state;         // look-back state of every pass: [pass][blocks][RADIX]
    unsigned int *tickets;       // one per pass
};

#ifndef GSB_HOST_EMU
extern __shared__ __align__(128) unsigned char gsb_sort_dynamic_smem[];
#endif

template <typename KeyT>
__global__ void __launch_bounds__(SORT_BLOCK_THREADS, GSB_SORT_MIN_BLOCKS)
onesweep_pass_kernel(const PassParams<KeyT> P) {
#ifdef GSB_HOST_EMU
    PassSmem<KeyT> &s = *reinterpret_cast<PassSmem<KeyT> *>(
        (reinterpret_cast<uintptr_t>(simt_emu::dynamic_smem()) + 127) & ~uintptr_t(127));
#else
    PassSmem<KeyT> &s = *reinterpret_cast<PassSmem<KeyT> *>(gsb_sort_dynamic_smem);
#endif
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    const int live = live_depth_bits(P.max_depth_key, P.depth_bits);
    const int npass = active_passes(P.end_bit, P.depth_bits, live);
    if (P.pass >= npass) return;  // surplus launch: the compacted key has fewer digits
    long long n = *P.n_dev;
    if (n > P.capacity) n = P.capacity;
    const DigitSel<KeyT> sel = make_digit_sel<KeyT>(P.pass, P.depth_bits, live);
    const bool to_b = ((npass - 1 - P.pass) & 1) == 0;
    const KeyT *const keys_in = P.pass == 0 ? P.keys_a : (to_b ? P.keys_c : P.keys_b);
    const int *const vals_in = P.pass == 0 ? P.vals_a : (to_b ? P.vals_c : P.vals_b);
    KeyT *const keys_out = to_b ? P.keys_b : P.keys_c;
    int *const vals_out = to_b ? P.vals_b : P.vals_c;
    const unsigned int *const hist = P.hist + P.pass * RADIX;
    unsigned int *const state = P.state + (size_t)P.pass * P.blocks * RADIX;
    if (tid == 0) mbar_init(&s.mbar, 1);
    unsigned int phase = 0;  // parity of the mbarrier phase the next bulk copy completes

    // The grid is as large as the GPU holds at once, not one CTA per key tile: a CTA sorts tile after tile in ticket order
    // until the frame's keys run out, so no CTA launches just to find that the frame has fewer keys than the capacity.
    // Look-back only waits on smaller tickets, which CTAs that are already running hold.
    for (;;) {
        if (tid == 0) s.ticket = atomicAdd(P.tickets + P.pass, 1u);
        {
            unsigned int *z = reinterpret_cast<unsigned int *>(&s.warp_cnt[0][0]);
#pragma unroll
            for (int i = 0; i < (SORT_BLOCK_THREADS / 32) * RADIX / 2 / SORT_BLOCK_THREADS; ++i) z[i * SORT_BLOCK_THREADS + tid] = 0;
        }
        __syncthreads();
        const unsigned int blk = s.ticket;
        const long long tile_base = (long long)blk * SORT_TILE;
        if (tile_base >= n) return;
        const int count = (int)min((long long)SORT_TILE, n - tile_base);

        // (a) key tile -> shared memory with one TMA bulk copy (16-byte granules); the < 16-byte tail of a
        //     partial last tile is fetched with ordinary loads.
        const unsigned int bulk_bytes = ((unsigned int)count * (unsigned int)sizeof(KeyT)) & ~15u;
        const int bulk_elems = (int)(bulk_bytes / sizeof(KeyT));
        if (tid == 0 && bulk_bytes) {
            fence_proxy_async_smem();  // the previous tile's reads of s.keys (ordered by the barrier above) come first
            mbar_arrive_expect_tx(&s.mbar, bulk_bytes);
            bulk_copy_g2s(s.keys, keys_in + tile_base, bulk_bytes, &s.mbar);
        }
        if (bulk_elems + tid < count) s.keys[bulk_elems + tid] = keys_in[tile_base + bulk_elems + tid];
        // payloads straight to registers, warp-striped (coalesced)
        int vals[SORT_ITEMS_PER_THREAD];
        const int wbase = warp * (32 * SORT_ITEMS_PER_THREAD);
        {
            const int *vp = vals_in + tile_base + wbase + lane;
#pragma unroll
            for (int j = 0; j < SORT_ITEMS_PER_THREAD; ++j)
                vals[j] = wbase + j * 32 + lane < count ? __ldg(vp + j * 32) : 0;
        }
        if (bulk_bytes) {
            mbar_wait(&s.mbar, phase);
            phase ^= 1u;
        }
        __syncthreads();  // tail keys written by other threads

        // (b) stable ranking: per-warp digit counters, match_digit groups equal digits in lane order
        KeyT keys[SORT_ITEMS_PER_THREAD];
        unsigned short ranks[SORT_ITEMS_PER_THREAD];
        const unsigned int lt_mask = (1u << lane) - 1u;
        unsigned short *const my_cnt = s.warp_cnt[warp];
#pragma unroll
        for (int j = 0; j < SORT_ITEMS_PER_THREAD; ++j) {
            const int idx = wbase + j * 32 + lane;
            const bool valid = idx < count;
            keys[j] = s.keys[idx];
            const int d = valid ? digit_of(keys[j], sel) : RADIX;
            const unsigned int peers = match_digit(d);
            unsigned int prev = 0;
            if (valid) prev = my_cnt[d];
            ranks[j] = (unsigned short)(prev + __popc(peers & lt_mask));
            __syncwarp();
            if (valid && (peers & lt_mask) == 0) my_cnt[d] = (unsigned short)(prev + __popc(peers));
            __syncwarp();
        }
        __syncthreads();

        // per-digit totals (thread t owns digit t), warp-exclusive bases; publish the aggregate at once
        unsigned int cnt = 0;
#pragma unroll
        for (int w = 0; w < SORT_BLOCK_THREADS / 32; ++w) {
            const unsigned int x = s.warp_cnt[w][tid];
            s.warp_cnt[w][tid] = (unsigned short)cnt;
            cnt += x;
        }
        unsigned int *const my_state = state + (size_t)blk * RADIX + tid;
        st_u32_volatile(my_state, (blk == 0 ? SS_INCLUSIVE : SS_AGGREGATE) | cnt);
        {   // block-exclusive digit starts
            unsigned int incl = cnt;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const unsigned int o = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) incl += o;
            }
            if (lane == 31) s.scan_tmp[warp] = incl;
            __syncthreads();
            unsigned int wprefix = 0;
#pragma unroll
            for (int w = 0; w < SORT_BLOCK_THREADS / 32; ++w)
                if (w < warp) wprefix += s.scan_tmp[w];
            s.digit_start[tid] = wprefix + incl - cnt;
        }
        const unsigned int dglobal = hist[tid];  // exclusive prefix over the digits of the whole array (histogram kernel)
        __syncthreads();  // digit_start and the warp bases are visible

        // block-sorted staging in shared memory (the TMA buffer is dead: all keys are in registers).  This needs
        // only block-local offsets, so it runs BEFORE the look-back and gives the predecessors time to publish.
#pragma unroll
        for (int j = 0; j < SORT_ITEMS_PER_THREAD; ++j) {
            const int idx = wbase + j * 32 + lane;
            if (idx < count) {
                const int d = digit_of(keys[j], sel);
                const unsigned int pos = s.digit_start[d] + my_cnt[d] + ranks[j];
                s.keys[pos] = keys[j];
                s.vals[pos] = vals[j];
            }
        }

        // (c) decoupled look-back over the preceding CTAs for this thread's digit, LOOKBACK predecessors in flight per round
        unsigned int excl = 0;
        if (blk != 0) {
            int look = (int)blk - 1;
            const unsigned int *const col = state + tid;
            bool done = false;
            while (!done) {
                unsigned int w[LOOKBACK];
#pragma unroll
                for (int r = 0; r < LOOKBACK; ++r)
                    w[r] = (look - r >= 0) ? ld_u32_volatile(col + (size_t)(look - r) * RADIX) : SS_INCLUSIVE;
#pragma unroll
                for (int r = 0; r < LOOKBACK; ++r) {
                    if (done) continue;
                    while ((w[r] >> 30) == 0) w[r] = ld_u32_volatile(col + (size_t)(look - r) * RADIX);
                    excl += w[r] & SS_VALUE_MASK;
                    done = (w[r] >> 30) == 2;
                }
                look -= LOOKBACK;
            }
            st_u32_volatile(my_state, SS_INCLUSIVE | (excl + cnt));
        }
        s.global_base[tid] = dglobal + excl - s.digit_start[tid];
        __syncthreads();

        // (d) scatter: consecutive local positions of one digit go to consecutive global addresses
#pragma unroll
        for (int j = 0; j < SORT_ITEMS_PER_THREAD; ++j) {
            const int pidx = j * SORT_BLOCK_THREADS + tid;
            if (pidx < count) {
                const KeyT k = s.keys[pidx];
                const unsigned int dst = s.global_base[digit_of(k, sel)] + (unsigned int)pidx;
                keys_out[dst] = k;
                vals_out[dst] = s.vals[pidx];
            }
        }
        __syncthreads();  // shared memory is free for the next tile
    }
}

#ifndef GSB_HOST_EMU
// in (never written) / out / tmp are three distinct buffers of `capacity` keys; `tickets` has one word per pass plus one
// (index 8) for the histogram kernel's completion count; `max_depth_key` may be NULL (no compaction).  `hist` and `tickets`
// must be zero; `state` need not be: the histogram kernel clears what the passes use.
template <typename KeyT>
static int sort_pairs_typed(const KeyT *keys_in, const int *vals_in, KeyT *keys_out, int *vals_out,
                            const long long *n_dev, int64_t capacity, int depth_bits, int end_bit,
                            const int *max_depth_key, unsigned int *hist, unsigned int *state, unsigned int *tickets,
                            KeyT *tmp_keys, int *tmp_vals, cudaStream_t stream) {
    const int passes = (end_bit + RBITS - 1) / RBITS;  // worst case: every depth bit live
    const int blocks = (int)((capacity + SORT_TILE - 1) / SORT_TILE);
    if (blocks == 0 || passes == 0) return GSB_OK;
    const size_t smem = sizeof(PassSmem<KeyT>);
    static int resident = 0;  // pass CTAs the whole GPU holds at once
    if (!resident) {
        GSB_CUDA_CHECK(cudaFuncSetAttribute(onesweep_pass_kernel<KeyT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            (int)smem));
        int per_sm = 0;
        GSB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, onesweep_pass_kernel<KeyT>,
                                                                     SORT_BLOCK_THREADS, smem));
        resident = (per_sm > 0 ? per_sm : 1) * num_sms();
    }
    const int pass_blocks = blocks < resident ? blocks : resident;
#ifndef GSB_HIST_BLOCKS_PER_SM
#define GSB_HIST_BLOCKS_PER_SM 4
#endif
    int hist_blocks = blocks < GSB_HIST_BLOCKS_PER_SM * num_sms() ? blocks : GSB_HIST_BLOCKS_PER_SM * num_sms();
    sort_histogram_kernel<KeyT><<<hist_blocks, SORT_BLOCK_THREADS, 0, stream>>>(keys_in, n_dev, capacity, depth_bits, end_bit,
                                                                                  max_depth_key, hist, tickets + 8, state,
                                                                                  (long long)blocks * RADIX);
    GSB_CUDA_CHECK(cudaGetLastError());
    PassParams<KeyT> P;
    P.keys_a = keys_in;
    P.vals_a = vals_in;
    P.keys_b = keys_out;
    P.vals_b = vals_out;
    P.keys_c = tmp_keys;
    P.vals_c = tmp_vals;
    P.n_dev = n_dev;
    P.capacity = capacity;
    P.depth_bits = depth_bits;
    P.end_bit = end_bit;
    P.blocks = blocks;
    P.max_depth_key = max_depth_key;
    P.hist = hist;
    P.state = state;
    P.tickets = tickets;
    for (int p = 0; p < passes; ++p) {
        P.pass = p;
        onesweep_pass_kernel<KeyT><<<pass_blocks, SORT_BLOCK_THREADS, smem, stream>>>(P);
        GSB_CUDA_CHECK(cudaGetLastError());
    }
    return GSB_OK;
}

int sort_pairs_device(const void *keys_in, const int *vals_in, void *keys_out, int *vals_out,
                      const long long *n_dev, int64_t n_capacity, int key_bytes, int depth_bits, int end_bit,
                      const int *max_depth_key, unsigned int *hist, unsigned int *state, unsigned int *tickets,
                      void *tmp_keys, int *tmp_vals, cudaStream_t stream) {
    typedef unsigned int u32;
    typedef unsigned long long u64;
    if (depth_bits < 0 || depth_bits > end_bit) {
        set_error("sort: depth_bits %d outside [0, end_bit = %d]", depth_bits, end_bit);
        return GSB_EINVAL;
    }
    if (key_bytes == 4)
        return sort_pairs_typed<u32>((const u32 *)keys_in, vals_in, (u32 *)keys_out, vals_out, n_dev, n_capacity, depth_bits,
                                     end_bit, max_depth_key, hist, state, tickets, (u32 *)tmp_keys, tmp_vals, stream);
    if (key_bytes == 8)
        return sort_pairs_typed<u64>((const u64 *)keys_in, vals_in, (u64 *)keys_out, vals_out, n_dev, n_capacity, depth_bits,
                                     end_bit, max_depth_key, hist, state, tickets, (u64 *)tmp_keys, tmp_vals, stream);
    set_error("sort: key_bytes must be 4 or 8, got %d", key_bytes);
    return GSB_EINVAL;
}

#endif  // GSB_HOST_EMU

// ------------------------------------------------------------------ tile ranges (GPCR:175-193)
template <typename KeyT>
__global__ void __launch_bounds__(256)
tile_ranges_kernel(const KeyT *__restrict__ keys, const long long *__restrict__ n_dev, long long capacity,
                   int depth_bits, int num_tiles, int *__restrict__ tile_start,
                   int *__restrict__ tile_end) {
    long long n = n_dev ? *n_dev : capacity;
    if (n > capacity) n = capacity;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const int t = (int)(keys[i] >> depth_bits);
        const int tp = i > 0 ? (int)(keys[i - 1] >> depth_bits) : -1;
        if (t != tp && t < num_tiles) {
            if (i > 0) {
                tile_start[t] = (int)i;
                if (tp < num_tiles) tile_end[tp] = (int)i;
            }
        }
        if (i == n - 1 && t < num_tiles) tile_end[t] = (int)n;
    }
}

#ifndef GSB_HOST_EMU
int launch_sort(const Workspace &ws, int64_t key_capacity, cudaStream_t stream) {
    const GsbWorkspaceLayout &L = ws.layout;
    // in = keys_a (emitted by the per-point kernel, never written), out = keys_b, scratch = keys_c; the number of passes
    // that actually run is decided on the device from the frame's largest depth key (CNT_MAX_DEPTH_KEY)
    (void)key_capacity;
    return sort_pairs_device(ws.keys_a, ws.vals_a, ws.keys_b, ws.vals_b, ws.counters + CNT_K, L.key_capacity_padded,
                             L.key_bytes, L.depth_bits, L.tile_bits + L.depth_bits,
                             reinterpret_cast<const int *>(ws.counters + CNT_MAX_DEPTH_KEY), ws.sort_hist, ws.sort_state,
                             ws.tickets + TICKET_SORT0, ws.keys_c, ws.vals_c, stream);
}

int launch_tile_ranges_raw(const long long *keys_i64, int64_t n, int *tile_start, int *tile_end,
                           int num_tiles, cudaStream_t stream) {
    if (n <= 0) return GSB_OK;
    long long blocks = (n + 255) / 256;
    const long long cap_blocks = 8LL * num_sms();
    if (blocks > cap_blocks) blocks = cap_blocks;
    tile_ranges_kernel<unsigned long long><<<(int)blocks, 256, 0, stream>>>(
        (const unsigned long long *)keys_i64, nullptr, n, 32, num_tiles, tile_start, tile_end);
    GSB_CUDA_CHECK(cudaGetLastError());
    return GSB_OK;
}

int launch_tile_ranges(const Workspace &ws, int64_t key_capacity, int num_tiles, cudaStream_t stream) {
    const GsbWorkspaceLayout &L = ws.layout;
    const void *keys = ws.keys_b;  // the sort always ends in b
    long long blocks = (key_capacity + 255) / 256;
    const long long cap_blocks = 8LL * num_sms();
    if (blocks > cap_blocks) blocks = cap_blocks;
    if (blocks <= 0) return GSB_OK;
    if (L.key_bytes == 4)
        tile_ranges_kernel<unsigned int><<<(int)blocks, 256, 0, stream>>>(
            (const unsigned int *)keys, ws.counters + CNT_K, key_capacity, L.depth_bits, num_tiles,
            ws.tile_start, ws.tile_end);
    else
        tile_ranges_kernel<unsigned long long><<<(int)blocks, 256, 0, stream>>>(
            (const unsigned long long *)keys, ws.counters + CNT_K, key_capacity, L.depth_bits, num_tiles,
            ws.tile_start, ws.tile_end);
    GSB_CUDA_CHECK(cudaGetLastError());
    return GSB_OK;
}

#endif  // GSB_HOST_EMU

}  // namespace gsb
