// emu_filter3d.cpp -- the 3D smoothing filter: the views kernels (csrc/filter3d.cu) launched as gsb200_filter3d_from_views
// launches them, and the FILTER instantiations of the per-point forward (csrc/preprocess.cu) and of the per-point backward
// (csrc/blend_bwd.cu, next to their unfiltered counterparts), compiled as host C++ under
// simt_emu.h.  TEST INFRASTRUCTURE, see simt_emu.h; a library of its own (tests/simt_filter3d_helpers.py).
#include "simt_emu.h"
// the kernel sources, unmodified (their launchers are compiled out under GSB_HOST_EMU)
#include "../../taichi_3d_gaussian_splatting_b200/csrc/preprocess.cu"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/filter3d.cu"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/blend_fwd.cu"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/blend_bwd.cu"

namespace gsb {
void set_error(const char *, ...) {}
}  // namespace gsb

extern "C" long long emu_filter3d_temp_bytes(int views, int objects) { return gsb::filter3d_temp_bytes(views, objects); }

// gsb200_filter3d_from_views after its argument checks: the pose blocks, the views kernel, the unseen-row kernel.  Returns the
// emulator's warp switches (> 0: the kernel ran its collectives).
extern "C" long long emu_filter3d_from_views(const GsbFilter3dViewsArgs *a) {
    using namespace gsb;
    simt_emu::M().switches = 0;
    const Filter3dParams p = filter3d_params(*a);
    *p.max_d_bits = 0;
    struct PoseArgs {
        const float *q, *t;
        int n;
        PoseBlock *out;
    } pa{a->q_pointcloud_camera, a->t_pointcloud_camera, (int)p.num_entries, const_cast<PoseBlock *>(p.poses)};
    simt_emu::launch([](const PoseArgs &x) { pose_kernel(x.q, x.t, x.n, x.out); }, (pa.n + 63) / 64, 64, pa);
    if (a->num_points > 0) {
        const int blocks = (int)((a->num_points + F3D_THREADS - 1) / F3D_THREADS);
        simt_emu::launch(filter3d_views_kernel, blocks, F3D_THREADS, p);
        simt_emu::launch(filter3d_unseen_kernel, blocks, F3D_THREADS, p);
    }
    return simt_emu::M().switches;
}

// preprocess_filter_kernel<unsigned int, GSB_LENS_PINHOLE> (filter3d != NULL) or preprocess_kernel<unsigned int> (NULL) on one
// frame with 32-bit keys: the records (12 N), point offsets and the counters
extern "C" long long emu_preprocess_filter(long long N, const float *xyz, float *features, const signed char *invalid,
                                           const int *obj_id, int n_obj, const float *q_pc, const float *t_pc, const float *K,
                                           int W, int H, float near_plane, float far_plane, float depth_scale, int depth_bits,
                                           long long key_capacity, long long *counters /*8*/, int *point_id, int *point_offset,
                                           int *num_tiles, float *records, float *point_in_camera, void *keys, int *vals,
                                           const float *filter3d) {
    using namespace gsb;
    std::vector<PoseBlock> poses(n_obj > 0 ? n_obj : 1);
    struct PoseArgs {
        const float *q, *t;
        int n;
        PoseBlock *out;
    } pa{q_pc, t_pc, n_obj, poses.data()};
    simt_emu::M().switches = 0;
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
    p.filter_tiles = 1;
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
    p.filter3d = filter3d;
    if (N > 0) {
        if (filter3d) simt_emu::launch(preprocess_filter_kernel<unsigned int, GSB_LENS_PINHOLE>, blocks, SCAN_BLOCK_THREADS, p);
        else simt_emu::launch(preprocess_kernel<unsigned int>, blocks, SCAN_BLOCK_THREADS, static_cast<const PreParams &>(p));
    }
    return simt_emu::M().switches;
}

// The per-point backward on given frame state (records, point_in_camera, accumulator rows, pose blocks), with the factors
// given: backward_points_filter_kernel<DEPTH, false> (filter3d != NULL) or backward_points_kernel<false, DEPTH> (NULL); with
// row_time != NULL the rolling-shutter pair backward_points_rs_filter_kernel<DEPTH, false> / backward_points_rs_kernel<DEPTH,
// false, false> with motion (6).  Grid as launch_backward_points_filter.

extern "C" void emu_backward_points_filter(long long N, const int *point_offset, const float *records, const float *point_in_camera,
                                           const float *accum, const float *poses, const float *xyz, const float *features,
                                           const int *obj_id, const float *t_pc_cam, const float *K, int color_max_sh_band,
                                           float q_f, float s_f, float a_f, float c_f, float h_f, float *grad_xyz,
                                           float *grad_feat, int depth, const float *filter3d, const float *motion,
                                           float *row_time) {
    using namespace gsb;
    PointsBwdRsFilterParams p;
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
    p.lens = LensParams();
    p.rs = RsParams();
    if (row_time) {
        for (int i = 0; i < 6; ++i) p.rs.motion[i] = motion[i];
        p.rs.row_time = row_time;
    }
    p.rs_partials = nullptr;
    p.filter3d = filter3d;
    long long blocks = N > 0 ? (N + GSB_POINTS_THREADS - 1) / GSB_POINTS_THREADS : 0;
    if (blocks > 16LL * 148) blocks = 16LL * 148;
    if (blocks <= 0) return;
    const int g = (int)blocks;
    if (row_time) {
        if (filter3d) {
            if (depth) simt_emu::launch(backward_points_rs_filter_kernel<true, false>, g, GSB_POINTS_THREADS, p);
            else simt_emu::launch(backward_points_rs_filter_kernel<false, false>, g, GSB_POINTS_THREADS, p);
        } else {
            const PointsBwdRsParams &q = p;
            if (depth) simt_emu::launch(backward_points_rs_kernel<true, false, false>, g, GSB_POINTS_THREADS, q);
            else simt_emu::launch(backward_points_rs_kernel<false, false, false>, g, GSB_POINTS_THREADS, q);
        }
    } else if (filter3d) {
        PointsBwdFilterParams f;
        static_cast<PointsBwdLensParams &>(f) = static_cast<const PointsBwdLensParams &>(p);
        f.filter3d = filter3d;
        if (depth) simt_emu::launch(backward_points_filter_kernel<true, false>, g, GSB_POINTS_THREADS, f);
        else simt_emu::launch(backward_points_filter_kernel<false, false>, g, GSB_POINTS_THREADS, f);
    } else {
        const PointsBwdParams &q = p;
        if (depth) simt_emu::launch(backward_points_kernel<false, true>, g, GSB_POINTS_THREADS, q);
        else simt_emu::launch(backward_points_kernel<false, false>, g, GSB_POINTS_THREADS, q);
    }
}
