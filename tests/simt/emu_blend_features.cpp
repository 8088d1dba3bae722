// emu_blend_features.cpp -- the feature-channel instantiations (gsb200_forward_ext / gsb200_backward_ext) of the forward blend
// and of loop A of the backward, alone and with the depth and alpha terms, compiled as host C++ under simt_emu.h.  TEST
// INFRASTRUCTURE, see simt_emu.h; built into its own library by tests/simt_feature_helpers.py with the same g++ flags as
// emu_blend.cpp (the other stages of the path come from that library, the per-point DEPTH kernel from emu_blend_depth.cpp).
#include "simt_emu.h"
// the kernel sources, unmodified (their launchers are compiled out under GSB_HOST_EMU)
#include "../../taichi_3d_gaussian_splatting_b200/csrc/blend_fwd.cu"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/blend_bwd.cu"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/blend_bwd_transposed.cu"

namespace gsb {
void set_error(const char *, ...) {}
}  // namespace gsb

// the channel count's compile-time width, as the launchers pick it
template <class F>
static void by_width(int C, F f) {
    if (C <= 4) f(std::integral_constant<int, 4>());
    else if (C <= 8) f(std::integral_constant<int, 8>());
    else f(std::integral_constant<int, 16>());
}

// blend_forward_kernel<false, EXACT_EXP, false, CF>: the full forward outputs plus the (H,W,C) feature map
extern "C" long long emu_blend_forward_features(int exact_exp, int H, int W, const int *tile_start, const int *tile_end,
                                                const int *sorted_vals, const float *records, const int *point_id, int C,
                                                const float *features, float *image, float *depth, float *acc_alpha,
                                                int *last_effective, int *valid_count, float *feature_map) {
    using namespace gsb;
    BlendFwdFeatParams p;
    p.H = H;
    p.W = W;
    p.tiles_x = W / GSB_TILE_WIDTH;
    p.tile_start = tile_start;
    p.tile_end = tile_end;
    p.sorted_vals = sorted_vals;
    p.records = reinterpret_cast<const float4 *>(records);
    p.image = image;
    p.depth = depth;
    p.acc_alpha = acc_alpha;
    p.last_effective = last_effective;
    p.valid_count = valid_count;
    p.work_counters = nullptr;
    p.channels = C;
    p.point_id = point_id;
    p.features = features;
    p.out_features = feature_map;
    const int tiles = p.tiles_x * (H / GSB_TILE_HEIGHT);
    simt_emu::M().switches = 0;
    by_width(C, [&](auto cf) {
        constexpr int CF = decltype(cf)::value;
        if (exact_exp) simt_emu::launch(blend_forward_kernel<false, true, false, CF>, tiles, GSB_TILE_PIXELS, p);
        else simt_emu::launch(blend_forward_kernel<false, false, false, CF>, tiles, GSB_TILE_PIXELS, p);
    });
    return simt_emu::M().switches;
}

template <bool EXACT_EXP, bool STATS, int CF>
static void launch_features(bool with_depth, bool with_alpha, int tiles, const gsb::BlendBwdFeatParams &p) {
    using gsb::blend_backward_transposed_kernel;
    if (with_depth && with_alpha)
        simt_emu::launch(blend_backward_transposed_kernel<EXACT_EXP, STATS, false, true, true, CF>, tiles, GSB_TILE_PIXELS, p);
    else if (with_depth)
        simt_emu::launch(blend_backward_transposed_kernel<EXACT_EXP, STATS, false, true, false, CF>, tiles, GSB_TILE_PIXELS, p);
    else if (with_alpha)
        simt_emu::launch(blend_backward_transposed_kernel<EXACT_EXP, STATS, false, false, true, CF>, tiles, GSB_TILE_PIXELS, p);
    else
        simt_emu::launch(blend_backward_transposed_kernel<EXACT_EXP, STATS, false, false, false, CF>, tiles, GSB_TILE_PIXELS, p);
}

// blend_backward_transposed_kernel<EXACT_EXP, STATS, false, DEPTH, ALPHA, CF>: grad_depth / depth non-null selects DEPTH,
// grad_alpha non-null ALPHA; grad_features (N,C) must be zero on entry (the library's call zeroes it)
extern "C" long long emu_blend_backward_features(int exact_exp, int stats, int H, int W, const int *tile_start,
                                                 const int *tile_end, const int *sorted_vals, const float *records,
                                                 const float *grad_image, const float *acc_alpha, const int *last_effective,
                                                 const float *grad_depth, const float *depth, const float *grad_alpha,
                                                 const int *point_id, int C, const float *features,
                                                 const float *grad_feature_map, float *grad_features, float *accum,
                                                 float *mag_image) {
    using namespace gsb;
    BlendBwdFeatParams p;
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
    p.feat = BlendFeatureParams{C, point_id, features, grad_feature_map, grad_features};
    const int tiles = p.tiles_x * (H / GSB_TILE_HEIGHT);
    simt_emu::M().switches = 0;
    const bool wd = grad_depth != nullptr, wa = grad_alpha != nullptr;
    by_width(C, [&](auto cf) {
        constexpr int CF = decltype(cf)::value;
        if (exact_exp) {
            if (stats) launch_features<true, true, CF>(wd, wa, tiles, p);
            else launch_features<true, false, CF>(wd, wa, tiles, p);
        } else {
            if (stats) launch_features<false, true, CF>(wd, wa, tiles, p);
            else launch_features<false, false, CF>(wd, wa, tiles, p);
        }
    });
    return simt_emu::M().switches;
}
