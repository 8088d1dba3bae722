// emu_blend_depth.cpp -- the depth-gradient instantiations (gsb200_backward_with_depth) of loop A of the backward and of the
// per-point chain rule, compiled as host C++ under simt_emu.h.  TEST INFRASTRUCTURE, see simt_emu.h; built into its own
// library by tests/simt_depth_helpers.py with the same g++ flags as emu_blend.cpp (the other stages of the path come from
// that library).
#include "simt_emu.h"
// the kernel sources, unmodified (their launchers are compiled out under GSB_HOST_EMU)
#include "../../taichi_3d_gaussian_splatting_b200/csrc/blend_fwd.cu"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/blend_bwd.cu"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/blend_bwd_transposed.cu"

namespace gsb {
void set_error(const char *, ...) {}
}  // namespace gsb

// blend_backward_transposed_kernel<EXACT_EXP, STATS, false, true>: grad_depth / depth are the (H,W) depth gradient and the
// forward's depth output
extern "C" long long emu_blend_backward_depth(int exact_exp, int stats, int H, int W, const int *tile_start, const int *tile_end,
                                              const int *sorted_vals, const float *records, const float *grad_image,
                                              const float *acc_alpha, const int *last_effective, const float *grad_depth,
                                              const float *depth, float *accum, float *mag_image) {
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
    const int tiles = p.tiles_x * (H / GSB_TILE_HEIGHT);
    simt_emu::M().switches = 0;
    if (exact_exp) {
        if (stats) simt_emu::launch(blend_backward_transposed_kernel<true, true, false, true>, tiles, GSB_TILE_PIXELS, p);
        else simt_emu::launch(blend_backward_transposed_kernel<true, false, false, true>, tiles, GSB_TILE_PIXELS, p);
    } else {
        if (stats) simt_emu::launch(blend_backward_transposed_kernel<false, true, false, true>, tiles, GSB_TILE_PIXELS, p);
        else simt_emu::launch(blend_backward_transposed_kernel<false, false, false, true>, tiles, GSB_TILE_PIXELS, p);
    }
    return simt_emu::M().switches;
}

// backward_points_kernel<COMPACT, true>: word 11 of the accumulator rows is dL/dz.  Same arguments as emu_backward_points
// (emu_blend.cpp); grad_sum / grad_col non-null selects the COMPACT instantiation.
extern "C" long long emu_backward_points_depth(long long N, const int *point_offset, const float *records,
                                               const float *point_in_camera, const float *accum, const float *poses,
                                               const float *xyz, const float *features, const int *obj_id,
                                               const float *t_pc_cam, const float *K, int color_max_sh_band, float q_f,
                                               float s_f, float a_f, float c_f, float h_f, float *grad_xyz, float *grad_feat,
                                               float *grad_sum, float *grad_col, int *ctl_num_in_camera, int *ctl_num_pixels,
                                               float *ctl_vs_grad, float *ctl_vs_grad_avg, float *ctl_pos_grad,
                                               float *ctl_pos_grad_norm) {
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
    p.grad_sum_compact = grad_sum;
    p.grad_color_compact = grad_col;
    p.ctl_num_in_camera = ctl_num_in_camera;
    p.ctl_num_pixels = ctl_num_pixels;
    p.ctl_vs_grad = ctl_vs_grad;
    p.ctl_vs_grad_avg = ctl_vs_grad_avg;
    p.ctl_pos_grad = ctl_pos_grad;
    p.ctl_pos_grad_norm = ctl_pos_grad_norm;
    p.skip_flag = nullptr;
    simt_emu::M().switches = 0;
    const int blocks = (int)std::min<long long>((N + GSB_POINTS_THREADS - 1) / GSB_POINTS_THREADS, 16 * 148);
    if (N > 0) {
        if (grad_sum) simt_emu::launch(backward_points_kernel<true, true>, blocks, GSB_POINTS_THREADS, p);
        else simt_emu::launch(backward_points_kernel<false, true>, blocks, GSB_POINTS_THREADS, p);
    }
    return simt_emu::M().switches;
}
