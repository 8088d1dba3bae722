// emu_blend_alpha.cpp -- the accumulated-alpha-gradient instantiations (gsb200_backward_aux with an alpha gradient) of loop A
// of the backward, alone and with the depth term, compiled as host C++ under simt_emu.h.  TEST INFRASTRUCTURE, see
// simt_emu.h; built into its own library by tests/simt_alpha_helpers.py with the same g++ flags as emu_blend.cpp (the
// other stages of the path come from that library, the per-point DEPTH kernel from emu_blend_depth.cpp).
#include "simt_emu.h"
// the kernel sources, unmodified (their launchers are compiled out under GSB_HOST_EMU)
#include "../../taichi_3d_gaussian_splatting_b200/csrc/blend_fwd.cu"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/blend_bwd.cu"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/blend_bwd_transposed.cu"

namespace gsb {
void set_error(const char *, ...) {}
}  // namespace gsb

template <bool EXACT_EXP, bool STATS>
static void launch_alpha(bool with_depth, int tiles, const gsb::BlendBwdParams &p) {
    using gsb::blend_backward_transposed_kernel;
    if (with_depth) simt_emu::launch(blend_backward_transposed_kernel<EXACT_EXP, STATS, false, true, true>, tiles, GSB_TILE_PIXELS, p);
    else simt_emu::launch(blend_backward_transposed_kernel<EXACT_EXP, STATS, false, false, true>, tiles, GSB_TILE_PIXELS, p);
}

// blend_backward_transposed_kernel<EXACT_EXP, STATS, false, DEPTH, true>: grad_alpha is the (H,W) gradient of the
// accumulated alpha; grad_depth / depth non-null selects the DEPTH + ALPHA instantiation
extern "C" long long emu_blend_backward_alpha(int exact_exp, int stats, int H, int W, const int *tile_start, const int *tile_end,
                                              const int *sorted_vals, const float *records, const float *grad_image,
                                              const float *acc_alpha, const int *last_effective, const float *grad_depth,
                                              const float *depth, const float *grad_alpha, float *accum, float *mag_image) {
    using namespace gsb;
    BlendBwdParams p;
    p.H = H;
    p.W = W;
    p.tiles_x = W / GSB_TILE_WIDTH;
    p.tile_start = tile_start;
    p.tile_end = tile_end;
    p.sorted_vals = sorted_vals;
    p.records = reinterpret_cast<const float4 *>(records);
    p.grad_image = grad_image;
    p.acc_alpha = acc_alpha;
    p.last_effective = last_effective;
    p.accum = accum;
    p.mag_image = mag_image;
    p.work_counters = nullptr;
    p.grad_depth = grad_depth;
    p.depth = depth;
    p.grad_alpha = grad_alpha;
    const int tiles = p.tiles_x * (H / GSB_TILE_HEIGHT);
    simt_emu::M().switches = 0;
    const bool with_depth = grad_depth != nullptr;
    if (exact_exp) {
        if (stats) launch_alpha<true, true>(with_depth, tiles, p);
        else launch_alpha<true, false>(with_depth, tiles, p);
    } else {
        if (stats) launch_alpha<false, true>(with_depth, tiles, p);
        else launch_alpha<false, false>(with_depth, tiles, p);
    }
    return simt_emu::M().switches;
}
