// emu_lens_grad.cpp -- the lens-coefficient gradient (gsb200_backward_lens_grad): the LGRAD instantiations of the per-point
// backward and the finishing kernel (csrc/blend_bwd.cu) and the coefficient helper of common.cuh, compiled as host C++ under
// simt_emu.h.  TEST INFRASTRUCTURE, see simt_emu.h; built into its own library by tests/simt_lens_grad_helpers.py with the same
// g++ flags as emu_blend.cpp (the lens forward and loop A come from the other emulator libraries).
#include "simt_emu.h"
// the kernel sources, unmodified (their launchers are compiled out under GSB_HOST_EMU)
#include "../../taichi_3d_gaussian_splatting_b200/csrc/blend_fwd.cu"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/blend_bwd.cu"

namespace gsb {
void set_error(const char *, ...) {}
}  // namespace gsb

// lens_coefficient_grad on n points: out (n, 5)
extern "C" void emu_lens_coefficient_grad(int model, long long n, const float *xn, const float *yn, const float *gx,
                                          const float *gy, const float *w00, const float *w01, const float *w11, float *out) {
    for (long long i = 0; i < n; ++i) {
        if (model == GSB_LENS_FISHEYE)
            gsb::lens_coefficient_grad<GSB_LENS_FISHEYE>(xn[i], yn[i], gx[i], gy[i], w00[i], w01[i], w11[i], out + 5 * i);
        else gsb::lens_coefficient_grad<GSB_LENS_OPENCV>(xn[i], yn[i], gx[i], gy[i], w00[i], w01[i], w11[i], out + 5 * i);
    }
}

// backward_points_lens_grad_kernel<DEPTH> on min(ceil(N/128), GSB_LENS_GRAD_PARTIAL_BLOCKS) CTAs as
// launch_backward_points_lens_grad, then lens_grad_finish_kernel: the dense gradients (no controller), the per-CTA partial
// rows (partials: GSB_LENS_GRAD_PARTIAL_BLOCKS * 5 floats) and the (5,) coefficient gradient.  Returns the grid size.
extern "C" int emu_backward_points_lens_grad(long long N, const int *point_offset, const float *records,
                                             const float *point_in_camera, const float *accum, const float *poses,
                                             const float *xyz, const float *features, const int *obj_id, const float *t_pc_cam,
                                             const float *K, int color_max_sh_band, float q_f, float s_f, float a_f, float c_f,
                                             float h_f, float *grad_xyz, float *grad_feat, int depth, int model,
                                             const float *coefficients, float *partials, float *grad_coefficients) {
    using namespace gsb;
    PointsBwdLensGradParams p;
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
    p.lens.model = model;
    for (int i = 0; i < 5; ++i) p.lens.k[i] = coefficients[i];
    p.lens.r2_max = (float)lens_r2_bound(model, coefficients);
    p.lens_partials = partials;
    const int blocks = (int)std::min<long long>(N > 0 ? (N + GSB_POINTS_THREADS - 1) / GSB_POINTS_THREADS : 0,
                                                GSB_LENS_GRAD_PARTIAL_BLOCKS);
    if (blocks > 0) {
        if (depth) simt_emu::launch(backward_points_lens_grad_kernel<true>, blocks, GSB_POINTS_THREADS, p);
        else simt_emu::launch(backward_points_lens_grad_kernel<false>, blocks, GSB_POINTS_THREADS, p);
    }
    struct FinishArgs {
        const float *partials;
        int blocks;
        float *g;
    } f{partials, blocks, grad_coefficients};
    simt_emu::launch([](const FinishArgs &a) { lens_grad_finish_kernel(a.partials, a.blocks, a.g); }, 1,
                     LENS_GRAD_FINISH_THREADS, f);
    return blocks;
}
