// emu_ortho.cpp -- the orthographic view (gsb200_forward_ortho / gsb200_backward_ortho): the per-point forward
// preprocess_ortho_kernel (csrc/preprocess.cu, with and without the 3D filter), the default instantiations of the forward blend
// and of the transposed loop A (the orthographic view does not change them), and the per-point backward
// backward_points_ortho_kernel with its pose and intrinsics finishing kernels (csrc/blend_bwd.cu), compiled as host C++ under
// simt_emu.h.  TEST INFRASTRUCTURE, see simt_emu.h; built into its own library by tests/simt_ortho_helpers.py with the same g++
// flags as emu_blend.cpp (the sort and the tile ranges come from that library).
#include "simt_emu.h"
// the kernel sources, unmodified (their launchers are compiled out under GSB_HOST_EMU)
#include "../../taichi_3d_gaussian_splatting_b200/csrc/preprocess.cu"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/blend_fwd.cu"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/blend_bwd.cu"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/blend_bwd_transposed.cu"

namespace gsb {
void set_error(const char *, ...) {}
}  // namespace gsb

// preprocess_ortho_kernel<KeyT, FILTER> on one frame (pose_kernel first, as launch_preprocess); filter3d NULL selects
// FILTER = false.  Returns the emulator's switch count.
extern "C" long long emu_preprocess_ortho(long long N, const float *xyz, float *features, const signed char *invalid,
                                          const int *obj_id, int n_obj, const float *q_pc, const float *t_pc, const float *K,
                                          int W, int H, float near_plane, float far_plane, float depth_scale, int depth_bits,
                                          int key_bytes, int filter_tiles, long long key_capacity, const float *filter3d,
                                          long long *counters /*8*/, int *point_id, int *point_offset, int *num_tiles,
                                          float *records /*12 N*/, float *point_in_camera /*3 N*/, void *keys, int *vals) {
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
    PreFilterParams p;
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
    p.lens = LensParams();
    p.lens.model = LENS_ORTHO;
    p.filter3d = filter3d;
    if (N > 0) {
        const bool f = filter3d != nullptr;
        if (key_bytes == 4) {
            if (f) simt_emu::launch(preprocess_ortho_kernel<unsigned int, true>, blocks, SCAN_BLOCK_THREADS, p);
            else simt_emu::launch(preprocess_ortho_kernel<unsigned int, false>, blocks, SCAN_BLOCK_THREADS, p);
        } else {
            if (f) simt_emu::launch(preprocess_ortho_kernel<unsigned long long, true>, blocks, SCAN_BLOCK_THREADS, p);
            else simt_emu::launch(preprocess_ortho_kernel<unsigned long long, false>, blocks, SCAN_BLOCK_THREADS, p);
        }
    }
    return simt_emu::M().switches;
}

template <class F>
static void by_width(int C, F f) {
    if (C <= 4) f(std::integral_constant<int, 4>());
    else if (C <= 8) f(std::integral_constant<int, 8>());
    else f(std::integral_constant<int, 16>());
}

// blend_forward_kernel<false, EXACT_EXP, false, CF>: the full outputs, plus the (H,W,C) feature map when C > 0
extern "C" long long emu_blend_forward_ortho(int exact_exp, int H, int W, const int *tile_start, const int *tile_end,
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
        if (exact_exp) simt_emu::launch(blend_forward_kernel<false, true, false, 0>, tiles, GSB_TILE_PIXELS, b);
        else simt_emu::launch(blend_forward_kernel<false, false, false, 0>, tiles, GSB_TILE_PIXELS, b);
    } else {
        by_width(C, [&](auto cf) {
            constexpr int CF = decltype(cf)::value;
            if (exact_exp) simt_emu::launch(blend_forward_kernel<false, true, false, CF>, tiles, GSB_TILE_PIXELS, p);
            else simt_emu::launch(blend_forward_kernel<false, false, false, CF>, tiles, GSB_TILE_PIXELS, p);
        });
    }
    return simt_emu::M().switches;
}

template <bool EXACT_EXP, bool STATS, int CF, class P>
static void launch_loop_a(bool with_depth, bool with_alpha, int tiles, const P &p) {
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

// blend_backward_transposed_kernel<true, false, false, DEPTH, ALPHA, CF>: grad_depth / depth non-null selects DEPTH,
// grad_alpha non-null ALPHA, C > 0 the feature width; grad_features (N,C) must be zero on entry
extern "C" long long emu_blend_backward_ortho(int H, int W, const int *tile_start, const int *tile_end, const int *sorted_vals,
                                              const float *records, const float *grad_image, const float *acc_alpha,
                                              const int *last_effective, const float *grad_depth, const float *depth,
                                              const float *grad_alpha, const int *point_id, int C, const float *features,
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
        launch_loop_a<true, false, 0>(wd, wa, tiles, b);
    } else {
        by_width(C, [&](auto cf) { launch_loop_a<true, false, decltype(cf)::value>(wd, wa, tiles, p); });
    }
    return simt_emu::M().switches;
}

// backward_points_ortho_kernel<DEPTH, POSE, INTR, FILTER> on the grid of launch_backward_points_ortho (pose or intr:
// min(ceil(N/128), GSB_POSE_PARTIAL_BLOCKS) CTAs; otherwise ceil(N/128) capped at 16 x 148), then pose_finish_kernel and
// intrinsics_finish_kernel as requested.  filter3d NULL selects FILTER = false.  Returns the grid size.
extern "C" int emu_backward_points_ortho(long long N, const int *point_offset, const float *records, const float *point_in_camera,
                                         const float *accum, const float *poses, const float *xyz, const float *features,
                                         const int *obj_id, const float *t_pc_cam, const float *K, int color_max_sh_band,
                                         float q_f, float s_f, float a_f, float c_f, float h_f, float *grad_xyz,
                                         float *grad_feat, int depth, const float *filter3d, int pose, int intr,
                                         int num_objects, const float *q_pc, float *pose_partials, float *grad_q,
                                         float *grad_t, float *intr_partials, float *grad_K) {
    using namespace gsb;
    PointsBwdOrthoParams p;
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
    p.pose_partials = pose ? pose_partials : nullptr;
    p.num_objects = pose ? num_objects : 0;
    p.intr_partials = intr ? intr_partials : nullptr;
    p.filter3d = filter3d;
    long long nb = N > 0 ? (N + GSB_POINTS_THREADS - 1) / GSB_POINTS_THREADS : 0;
    const long long cap = (pose || intr) ? (long long)GSB_POSE_PARTIAL_BLOCKS : 16LL * 148;
    const int blocks = (int)std::min(nb, cap);
    const int mode = filter3d ? 4 : pose && intr ? 3 : pose ? 2 : intr ? 1 : 0;
    auto run = [&](auto dep) {
        constexpr bool D = decltype(dep)::value;
        if (mode == 4) simt_emu::launch(backward_points_ortho_kernel<D, false, false, true>, blocks, GSB_POINTS_THREADS, p);
        else if (mode == 3) simt_emu::launch(backward_points_ortho_kernel<D, true, true, false>, blocks, GSB_POINTS_THREADS, p);
        else if (mode == 2) simt_emu::launch(backward_points_ortho_kernel<D, true, false, false>, blocks, GSB_POINTS_THREADS, p);
        else if (mode == 1) simt_emu::launch(backward_points_ortho_kernel<D, false, true, false>, blocks, GSB_POINTS_THREADS, p);
        else simt_emu::launch(backward_points_ortho_kernel<D, false, false, false>, blocks, GSB_POINTS_THREADS, p);
    };
    if (blocks > 0) {
        if (depth) run(std::true_type());
        else run(std::false_type());
    }
    if (pose) {
        struct FinishArgs {
            const float *partials;
            int blocks, num_objects;
            const float *q, *t;
            float *gq, *gt;
        } f{pose_partials, blocks, num_objects, q_pc, t_pc_cam, grad_q, grad_t};
        simt_emu::launch(
            [](const FinishArgs &a) { pose_finish_kernel(a.partials, a.blocks, a.num_objects, a.q, a.t, a.gq, a.gt); },
            num_objects, POSE_FINISH_THREADS, f);
    }
    if (intr) {
        struct IntrFinishArgs {
            const float *partials;
            int blocks;
            float *gK;
        } fi{intr_partials, blocks, grad_K};
        simt_emu::launch([](const IntrFinishArgs &a) { intrinsics_finish_kernel(a.partials, a.blocks, a.gK); }, 1,
                         INTR_FINISH_THREADS, fi);
    }
    return blocks;
}
