// emu_equirect.cpp -- the equirectangular panorama (gsb200_forward_equirect / gsb200_backward_equirect): the per-point
// forward preprocess_equirect_kernel (csrc/preprocess.cu), the WRAP instantiations of the forward blend and of the transposed
// loop A, and the per-point backward backward_points_equirect_kernel (csrc/blend_bwd.cu), compiled as host C++ under
// simt_emu.h.  TEST INFRASTRUCTURE, see simt_emu.h; built into its own library by tests/simt_equirect_helpers.py with the
// same g++ flags as emu_blend.cpp (the sort and the tile ranges come from that library: the panorama does not change them).
#include "simt_emu.h"
// the kernel sources, unmodified (their launchers are compiled out under GSB_HOST_EMU)
#include "../../taichi_3d_gaussian_splatting_b200/csrc/preprocess.cu"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/blend_fwd.cu"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/blend_bwd.cu"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/blend_bwd_transposed.cu"

namespace gsb {
void set_error(const char *, ...) {}
}  // namespace gsb

// preprocess_equirect_kernel<KeyT> on one frame (pose_kernel first, as launch_preprocess); returns the emulator's switch count
extern "C" long long emu_preprocess_equirect(long long N, const float *xyz, float *features, const signed char *invalid,
                                             const int *obj_id, int n_obj, const float *q_pc, const float *t_pc, const float *K,
                                             int W, int H, float near_plane, float far_plane, float depth_scale, int depth_bits,
                                             int key_bytes, int filter_tiles, long long key_capacity, long long *counters /*8*/,
                                             int *point_id, int *point_offset, int *num_tiles, float *records /*12 N*/,
                                             float *point_in_camera /*3 N*/, void *keys, int *vals) {
    using namespace gsb;
    std::vector<PoseBlock> poses(n_obj > 0 ? n_obj : 1);
    struct PoseArgs {
        const float *q, *t;
        int n;
        PoseBlock *out;
    } pa{q_pc, t_pc, n_obj, poses.data()};
    simt_emu::M().switches = 0;
    if (n_obj > 0)
        simt_emu::launch([](const PoseArgs &a) { pose_kernel(a.q, a.t, a.n, a.out); }, (n_obj + 63) / 64, 64, pa);
    const int blocks = (int)((N + SCAN_BLOCK_THREADS - 1) / SCAN_BLOCK_THREADS);
    std::vector<unsigned int> tickets(16, 0u);
    std::vector<unsigned long long> scan_state(blocks + 1, 0ull);
    PreParams p;
    p.N = N;
    p.xyz = xyz;
    p.features = features;
    p.invalid = invalid;
    p.obj_id = obj_id;
    p.poses = poses.data();
    p.K = K;
    p.W = W;
    p.H = H;
    p.near_plane = near_plane;
    p.far_plane = far_plane;
    p.depth_scale = depth_scale;
    p.depth_bits = depth_bits;
    p.skip_q_normalise = 0;
    p.filter_tiles = filter_tiles;
    p.key_capacity = key_capacity;
    p.key_store_limit = key_capacity;
    p.num_blocks = blocks;
    p.counters = counters;
    p.tickets = tickets.data();
    p.scan_state = scan_state.data();
    p.point_id = point_id;
    p.point_offset = point_offset;
    p.num_tiles = num_tiles;
    p.records = reinterpret_cast<float4 *>(records);
    p.point_in_camera = point_in_camera;
    p.keys = keys;
    p.vals = vals;
    if (N > 0) {
        if (key_bytes == 4) simt_emu::launch(preprocess_equirect_kernel<unsigned int>, blocks, SCAN_BLOCK_THREADS, p);
        else simt_emu::launch(preprocess_equirect_kernel<unsigned long long>, blocks, SCAN_BLOCK_THREADS, p);
    }
    return simt_emu::M().switches;
}

template <class F>
static void by_width(int C, F f) {
    if (C <= 4) f(std::integral_constant<int, 4>());
    else if (C <= 8) f(std::integral_constant<int, 8>());
    else f(std::integral_constant<int, 16>());
}

// blend_forward_kernel<false, EXACT_EXP, false, CF, true>: the full outputs, plus the (H,W,C) feature map when C > 0
extern "C" long long emu_blend_forward_equirect(int exact_exp, int H, int W, const int *tile_start, const int *tile_end,
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
    if (C == 0) {
        const BlendFwdParams &b = p;
        if (exact_exp) simt_emu::launch(blend_forward_kernel<false, true, false, 0, true>, tiles, GSB_TILE_PIXELS, b);
        else simt_emu::launch(blend_forward_kernel<false, false, false, 0, true>, tiles, GSB_TILE_PIXELS, b);
    } else {
        by_width(C, [&](auto cf) {
            constexpr int CF = decltype(cf)::value;
            if (exact_exp) simt_emu::launch(blend_forward_kernel<false, true, false, CF, true>, tiles, GSB_TILE_PIXELS, p);
            else simt_emu::launch(blend_forward_kernel<false, false, false, CF, true>, tiles, GSB_TILE_PIXELS, p);
        });
    }
    return simt_emu::M().switches;
}

template <bool EXACT_EXP, bool STATS, int CF, class P>
static void launch_loop_a(bool with_depth, bool with_alpha, int tiles, const P &p) {
    using gsb::blend_backward_transposed_kernel;
    if (with_depth && with_alpha)
        simt_emu::launch(blend_backward_transposed_kernel<EXACT_EXP, STATS, false, true, true, CF, true>, tiles, GSB_TILE_PIXELS, p);
    else if (with_depth)
        simt_emu::launch(blend_backward_transposed_kernel<EXACT_EXP, STATS, false, true, false, CF, true>, tiles, GSB_TILE_PIXELS, p);
    else if (with_alpha)
        simt_emu::launch(blend_backward_transposed_kernel<EXACT_EXP, STATS, false, false, true, CF, true>, tiles, GSB_TILE_PIXELS, p);
    else
        simt_emu::launch(blend_backward_transposed_kernel<EXACT_EXP, STATS, false, false, false, CF, true>, tiles, GSB_TILE_PIXELS, p);
}

template <int CF, class P>
static void launch_loop_a_flags(bool exact, bool stats, bool wd, bool wa, int tiles, const P &p) {
    if (exact) {
        if (stats) launch_loop_a<true, true, CF>(wd, wa, tiles, p);
        else launch_loop_a<true, false, CF>(wd, wa, tiles, p);
    } else {
        if (stats) launch_loop_a<false, true, CF>(wd, wa, tiles, p);
        else launch_loop_a<false, false, CF>(wd, wa, tiles, p);
    }
}

// blend_backward_transposed_kernel<EXACT_EXP, STATS, false, DEPTH, ALPHA, CF, true>: grad_depth / depth non-null selects DEPTH,
// grad_alpha non-null ALPHA, C > 0 the feature width; grad_features (N,C) must be zero on entry
extern "C" long long emu_blend_backward_equirect(int exact_exp, int stats, int H, int W, const int *tile_start,
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
    if (C == 0) {
        const BlendBwdParams &b = p;
        launch_loop_a_flags<0>(exact_exp != 0, stats != 0, wd, wa, tiles, b);
    } else {
        by_width(C, [&](auto cf) { launch_loop_a_flags<decltype(cf)::value>(exact_exp != 0, stats != 0, wd, wa, tiles, p); });
    }
    return simt_emu::M().switches;
}

// backward_points_equirect_kernel<DEPTH> on the grid of launch_backward_points_equirect: the dense gradients (no controller)
extern "C" void emu_backward_points_equirect(long long N, const int *point_offset, const float *records, const float *point_in_camera,
                                             const float *accum, const float *poses, const float *xyz, const float *features,
                                             const int *obj_id, const float *t_pc_cam, const float *K, int color_max_sh_band,
                                             float q_f, float s_f, float a_f, float c_f, float h_f, float *grad_xyz,
                                             float *grad_feat, int depth) {
    using namespace gsb;
    PointsBwdParams p;
    p.N = N;
    p.point_offset = point_offset;
    p.records = reinterpret_cast<const float4 *>(records);
    p.point_in_camera = point_in_camera;
    p.accum = accum;
    p.poses = reinterpret_cast<const PoseBlock *>(poses);
    p.xyz = xyz;
    p.features = features;
    p.obj_id = obj_id;
    p.t_pc_cam = t_pc_cam;
    p.K = K;
    const int band = color_max_sh_band;
    p.first_cleared = band <= 0 ? 1 : band == 1 ? 4 : band == 2 ? 9 : 16;  // as launch_backward_points
    p.q_f = q_f;
    p.s_f = s_f;
    p.a_f = a_f;
    p.c_f = c_f;
    p.h_f = h_f;
    p.grad_xyz = grad_xyz;
    p.grad_feat = grad_feat;
    p.grad_sum_compact = nullptr;
    p.grad_color_compact = nullptr;
    p.ctl_num_in_camera = nullptr;
    p.ctl_num_pixels = nullptr;
    p.ctl_vs_grad = nullptr;
    p.ctl_vs_grad_avg = nullptr;
    p.ctl_pos_grad = nullptr;
    p.ctl_pos_grad_norm = nullptr;
    p.skip_flag = nullptr;
    long long blocks = N > 0 ? (N + GSB_POINTS_THREADS - 1) / GSB_POINTS_THREADS : 0;
    if (blocks > 16LL * 148) blocks = 16LL * 148;
    if (blocks <= 0) return;
    if (depth) simt_emu::launch(backward_points_equirect_kernel<true>, (int)blocks, GSB_POINTS_THREADS, p);
    else simt_emu::launch(backward_points_equirect_kernel<false>, (int)blocks, GSB_POINTS_THREADS, p);
}
