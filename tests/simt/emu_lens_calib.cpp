// emu_lens_calib.cpp -- pose and intrinsics gradients through a lens (gsb200_backward_lens_calib): the LENS instantiations of
// the per-point backward with pose / intrinsics / coefficient sums and their finishing kernels (csrc/blend_bwd.cu), compiled as
// host C++ under simt_emu.h.  TEST INFRASTRUCTURE, see simt_emu.h; built into its own library by
// tests/simt_lens_calib_helpers.py with the same g++ flags as emu_blend.cpp (the lens forward and loop A come from the other
// emulator libraries).
#include "simt_emu.h"
// the kernel sources, unmodified (their launchers are compiled out under GSB_HOST_EMU)
#include "../../taichi_3d_gaussian_splatting_b200/csrc/blend_fwd.cu"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/blend_bwd.cu"

namespace gsb {
void set_error(const char *, ...) {}
}  // namespace gsb

template <bool DEPTH>
static void run_kernel(bool pose, bool intr, bool lgrad, int blocks, const gsb::PointsBwdLensCalibParams &p) {
    using namespace gsb;
    if (pose && intr && lgrad) simt_emu::launch(backward_points_lens_calib_kernel<DEPTH, true, true, true>, blocks, GSB_POINTS_THREADS, p);
    else if (pose && intr) simt_emu::launch(backward_points_lens_calib_kernel<DEPTH, true, true, false>, blocks, GSB_POINTS_THREADS, p);
    else if (pose && lgrad) simt_emu::launch(backward_points_lens_calib_kernel<DEPTH, true, false, true>, blocks, GSB_POINTS_THREADS, p);
    else if (pose) simt_emu::launch(backward_points_lens_calib_kernel<DEPTH, true, false, false>, blocks, GSB_POINTS_THREADS, p);
    else if (lgrad) simt_emu::launch(backward_points_lens_calib_kernel<DEPTH, false, true, true>, blocks, GSB_POINTS_THREADS, p);
    else simt_emu::launch(backward_points_lens_calib_kernel<DEPTH, false, true, false>, blocks, GSB_POINTS_THREADS, p);
}

// backward_points_lens_calib_kernel<DEPTH, POSE, INTR, LGRAD> on min(ceil(N/128), GSB_POSE_PARTIAL_BLOCKS) CTAs as
// launch_backward_points_lens_calib (pose or intr must be set), then pose_finish_kernel (pose), intrinsics_finish_kernel
// (intr) and lens_grad_finish_kernel (lgrad): the dense gradients (no controller), the per-CTA partial rows (as the
// emulators of the pose, intrinsics and coefficient gradients) and the (K,4) / (K,3) pose, (3,3) K and (5,) coefficient
// gradients of the sums that are on.  Returns the grid size.
extern "C" int emu_backward_points_lens_calib(long long N, const int *point_offset, const float *records,
                                              const float *point_in_camera, const float *accum, const float *poses,
                                              const float *xyz, const float *features, const int *obj_id, const float *t_pc_cam,
                                              const float *K, int color_max_sh_band, float q_f, float s_f, float a_f, float c_f,
                                              float h_f, float *grad_xyz, float *grad_feat, int depth, int model,
                                              const float *coefficients, int pose, int intr, int lgrad, int num_objects,
                                              const float *q_pc, float *pose_partials, float *grad_q, float *grad_t,
                                              float *intr_partials, float *grad_K, float *lens_partials,
                                              float *grad_coefficients) {
    using namespace gsb;
    PointsBwdLensCalibParams p;
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
    p.lens.model = model;
    for (int i = 0; i < 5; ++i) p.lens.k[i] = coefficients[i];
    p.lens.r2_max = (float)lens_r2_bound(model, coefficients);
    p.lens_partials = lgrad ? lens_partials : nullptr;
    const int blocks = (int)std::min<long long>(N > 0 ? (N + GSB_POINTS_THREADS - 1) / GSB_POINTS_THREADS : 0,
                                                GSB_POSE_PARTIAL_BLOCKS);
    if (blocks > 0) {
        if (depth) run_kernel<true>(pose != 0, intr != 0, lgrad != 0, blocks, p);
        else run_kernel<false>(pose != 0, intr != 0, lgrad != 0, blocks, p);
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
    struct RowFinishArgs {
        const float *partials;
        int blocks;
        float *g;
    };
    if (intr) {
        RowFinishArgs fi{intr_partials, blocks, grad_K};
        simt_emu::launch([](const RowFinishArgs &a) { intrinsics_finish_kernel(a.partials, a.blocks, a.g); }, 1,
                         INTR_FINISH_THREADS, fi);
    }
    if (lgrad) {
        RowFinishArgs fl{lens_partials, blocks, grad_coefficients};
        simt_emu::launch([](const RowFinishArgs &a) { lens_grad_finish_kernel(a.partials, a.blocks, a.g); }, 1,
                         LENS_GRAD_FINISH_THREADS, fl);
    }
    return blocks;
}
