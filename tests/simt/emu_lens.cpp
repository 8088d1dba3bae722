// emu_lens.cpp -- lens distortion (gsb200_forward_lens / gsb200_backward_lens): the lens instantiations of the per-point
// forward (csrc/preprocess.cu) and of the per-point backward (csrc/blend_bwd.cu), the lens helper and the host bound of
// common.cuh, compiled as host C++ under simt_emu.h.  TEST INFRASTRUCTURE, see simt_emu.h; built into its own library by
// tests/simt_lens_helpers.py with the same g++ flags as emu_blend.cpp (sort, tile ranges, forward blend and loop A come from
// the other emulator libraries: the lens does not change them).
#include "simt_emu.h"
// the kernel sources, unmodified (their launchers are compiled out under GSB_HOST_EMU)
#include "../../taichi_3d_gaussian_splatting_b200/csrc/preprocess.cu"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/blend_fwd.cu"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/blend_bwd.cu"

namespace gsb {
void set_error(const char *, ...) {}
}  // namespace gsb

static gsb::LensParams make_lens(int model, const float *coefficients) {
    gsb::LensParams l;
    l.model = model;
    for (int i = 0; i < 5; ++i) l.k[i] = coefficients[i];
    l.r2_max = (float)gsb::lens_r2_bound(model, coefficients);
    return l;
}

// the r^2 bound the library passes to the kernels (host, double)
extern "C" double emu_lens_r2_bound(int model, const float *coefficients) { return gsb::lens_r2_bound(model, coefficients); }

// lens_distort on n points: the displacement (ox, oy) = (xd - xn, yd - yn) and D (row-major 2x2) per point
extern "C" void emu_lens_distort(int model, const float *coefficients, long long n, const float *xn, const float *yn, float *ox,
                                 float *oy, float *D) {
    for (long long i = 0; i < n; ++i) {
        if (model == GSB_LENS_FISHEYE) gsb::lens_distort<GSB_LENS_FISHEYE>(coefficients, xn[i], yn[i], ox[i], oy[i], D + 4 * i);
        else gsb::lens_distort<GSB_LENS_OPENCV>(coefficients, xn[i], yn[i], ox[i], oy[i], D + 4 * i);
    }
}

// emu_preprocess (emu_preprocess.cpp) with preprocess_lens_kernel<KeyT, model>; model is GSB_LENS_OPENCV or GSB_LENS_FISHEYE
extern "C" long long emu_preprocess_lens(long long N, const float *xyz, float *features, const signed char *invalid,
                                         const int *obj_id, int n_obj, const float *q_pc, const float *t_pc, const float *K,
                                         int W, int H, float near_plane, float far_plane, float depth_scale, int depth_bits,
                                         int key_bytes, int filter_tiles, int skip_q_normalise, long long key_capacity,
                                         long long *counters /*8*/, int *point_id, int *point_offset, int *num_tiles,
                                         float *records /*12 N*/, float *point_in_camera /*3 N*/, void *keys, int *vals,
                                         int model, const float *coefficients) {
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
    PreLensParams p;
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
    p.skip_q_normalise = skip_q_normalise;
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
    p.lens = make_lens(model, coefficients);
    if (N > 0) {
        const bool fisheye = model == GSB_LENS_FISHEYE;
        if (key_bytes == 4) {
            if (fisheye) simt_emu::launch(preprocess_lens_kernel<unsigned int, GSB_LENS_FISHEYE>, blocks, SCAN_BLOCK_THREADS, p);
            else simt_emu::launch(preprocess_lens_kernel<unsigned int, GSB_LENS_OPENCV>, blocks, SCAN_BLOCK_THREADS, p);
        } else {
            if (fisheye) simt_emu::launch(preprocess_lens_kernel<unsigned long long, GSB_LENS_FISHEYE>, blocks, SCAN_BLOCK_THREADS, p);
            else simt_emu::launch(preprocess_lens_kernel<unsigned long long, GSB_LENS_OPENCV>, blocks, SCAN_BLOCK_THREADS, p);
        }
    }
    return simt_emu::M().switches;
}

// backward_points_lens_kernel<DEPTH> on the grid of launch_backward_points_lens: the dense gradients (no controller)
extern "C" long long emu_backward_points_lens(long long N, const int *point_offset, const float *records,
                                              const float *point_in_camera, const float *accum, const float *poses,
                                              const float *xyz, const float *features, const int *obj_id, const float *t_pc_cam,
                                              const float *K, int color_max_sh_band, float q_f, float s_f, float a_f, float c_f,
                                              float h_f, float *grad_xyz, float *grad_feat, int depth, int model,
                                              const float *coefficients) {
    using namespace gsb;
    PointsBwdLensParams p;
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
    p.lens = make_lens(model, coefficients);
    simt_emu::M().switches = 0;
    const int blocks = (int)std::min<long long>((N + GSB_POINTS_THREADS - 1) / GSB_POINTS_THREADS, 16 * 148);
    if (N > 0) {
        if (depth) simt_emu::launch(backward_points_lens_kernel<true>, blocks, GSB_POINTS_THREADS, p);
        else simt_emu::launch(backward_points_lens_kernel<false>, blocks, GSB_POINTS_THREADS, p);
    }
    return simt_emu::M().switches;
}
