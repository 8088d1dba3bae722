// emu_defocus.cpp -- the depth of field (gsb200_forward_defocus / gsb200_backward_defocus): the DEFOCUS instantiations of the
// per-point forward (csrc/preprocess.cu), of the per-point backward and the finishing kernel (csrc/blend_bwd.cu), with and
// without a lens, a rolling shutter and motion blur, compiled as host C++ under simt_emu.h.  TEST INFRASTRUCTURE, see
// simt_emu.h; built into its own library by tests/simt_defocus_helpers.py with the same g++ flags as emu_blend.cpp (sort,
// tile ranges, forward blend and loop A come from the other emulator libraries: the defocus does not change them).
#include "simt_emu.h"
// the kernel sources, unmodified (their launchers are compiled out under GSB_HOST_EMU)
#include "../../taichi_3d_gaussian_splatting_b200/csrc/preprocess.cu"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/blend_fwd.cu"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/blend_bwd.cu"

namespace gsb {
void set_error(const char *, ...) {}
}  // namespace gsb

// model GSB_LENS_PINHOLE: no lens (the coefficients are ignored)
static gsb::LensParams make_lens(int model, const float *coefficients) {
    gsb::LensParams l;
    l.model = model;
    for (int i = 0; i < 5; ++i) l.k[i] = model == GSB_LENS_PINHOLE ? 0.0f : coefficients[i];
    l.r2_max = (float)gsb::lens_r2_bound(model, l.k);
    return l;
}

static gsb::RsParams make_rs(const float *motion, float *row_time) {
    gsb::RsParams r;
    for (int i = 0; i < 6; ++i) r.motion[i] = motion[i];
    r.row_time = row_time;
    return r;
}

template <typename KeyT>
static void launch_defocus_pre(int model, bool rolling, int blocks, const gsb::PreBlurParams &p) {
    using namespace gsb;
    if (rolling) {
        if (model == GSB_LENS_FISHEYE) simt_emu::launch(preprocess_blur_kernel<KeyT, GSB_LENS_FISHEYE, true, true>, blocks, SCAN_BLOCK_THREADS, p);
        else if (model == GSB_LENS_OPENCV) simt_emu::launch(preprocess_blur_kernel<KeyT, GSB_LENS_OPENCV, true, true>, blocks, SCAN_BLOCK_THREADS, p);
        else simt_emu::launch(preprocess_blur_kernel<KeyT, GSB_LENS_PINHOLE, true, true>, blocks, SCAN_BLOCK_THREADS, p);
    } else {
        if (model == GSB_LENS_FISHEYE) simt_emu::launch(preprocess_blur_kernel<KeyT, GSB_LENS_FISHEYE, false, true>, blocks, SCAN_BLOCK_THREADS, p);
        else if (model == GSB_LENS_OPENCV) simt_emu::launch(preprocess_blur_kernel<KeyT, GSB_LENS_OPENCV, false, true>, blocks, SCAN_BLOCK_THREADS, p);
        else simt_emu::launch(preprocess_blur_kernel<KeyT, GSB_LENS_PINHOLE, false, true>, blocks, SCAN_BLOCK_THREADS, p);
    }
}

// emu_preprocess_blur (emu_motion_blur.cpp) with preprocess_blur_kernel<KeyT, model, rolling, true> and the thin lens
// defocus = (a, rho) beside the exposure motion `blur` (zeros: none); row_time (N) is written with `rolling`
extern "C" long long emu_preprocess_defocus(long long N, const float *xyz, float *features, const signed char *invalid,
                                       const int *obj_id, int n_obj, const float *q_pc, const float *t_pc, const float *K, int W,
                                       int H, float near_plane, float far_plane, float depth_scale, int depth_bits, int key_bytes,
                                       int filter_tiles, int skip_q_normalise, long long key_capacity, long long *counters /*8*/,
                                       int *point_id, int *point_offset, int *num_tiles, float *records /*12 N*/,
                                       float *point_in_camera /*3 N*/, void *keys, int *vals, int model, const float *coefficients,
                                       const float *motion, float *row_time, int rolling, const float *blur,
                                       const float *defocus) {
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
    PreBlurParams p;
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
    p.rs = make_rs(motion, row_time);
    for (int i = 0; i < 6; ++i) p.blur.motion[i] = blur[i];
    p.defocus.aperture = defocus[0];
    p.defocus.inverse_focus = defocus[1];
    if (N > 0) {
        if (key_bytes == 4) launch_defocus_pre<unsigned int>(model, rolling != 0, blocks, p);
        else launch_defocus_pre<unsigned long long>(model, rolling != 0, blocks, p);
    }
    return simt_emu::M().switches;
}

template <bool DEPTH, bool LENS, bool RS>
static void launch_defocus(bool dgrad, int blocks, const gsb::PointsBwdBlurParams &p) {
    if (dgrad) simt_emu::launch(gsb::backward_points_blur_kernel<DEPTH, LENS, RS, false, true, true>, blocks, GSB_POINTS_THREADS, p);
    else simt_emu::launch(gsb::backward_points_blur_kernel<DEPTH, LENS, RS, false, true, false>, blocks, GSB_POINTS_THREADS, p);
}
template <bool DEPTH, bool LENS>
static void launch_defocus_rs(bool rolling, bool dgrad, int blocks, const gsb::PointsBwdBlurParams &p) {
    if (rolling) launch_defocus<DEPTH, LENS, true>(dgrad, blocks, p);
    else launch_defocus<DEPTH, LENS, false>(dgrad, blocks, p);
}

// backward_points_blur_kernel<DEPTH, LENS, RS, false, true, DGRAD> on the grid of launch_backward_points_blur (LENS = model !=
// pinhole, RS = rolling): the dense gradients (no controller); with dgrad also the per-CTA rows (partials:
// (GSB_RS_GRAD_PARTIAL_BLOCKS + 1) * 6 floats, the finished row last) and, after rolling_shutter_grad_finish_kernel, the (2,)
// defocus gradient, its first two values.  Returns the grid size.
extern "C" int emu_backward_points_defocus(long long N, const int *point_offset, const float *records, const float *point_in_camera,
                                      const float *accum, const float *poses, const float *xyz, const float *features,
                                      const int *obj_id, const float *t_pc_cam, const float *K, int color_max_sh_band, float q_f,
                                      float s_f, float a_f, float c_f, float h_f, float *grad_xyz, float *grad_feat, int depth,
                                      int model, const float *coefficients, const float *motion, float *row_time, int rolling,
                                      const float *blur, const float *defocus, int mgrad, float *partials,
                                      float *grad_defocus) {
    using namespace gsb;
    PointsBwdBlurParams p;
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
    p.rs = make_rs(motion, row_time);
    p.rs_partials = partials;
    for (int i = 0; i < 6; ++i) p.blur.motion[i] = blur[i];
    p.defocus.aperture = defocus[0];
    p.defocus.inverse_focus = defocus[1];
    long long blocks = N > 0 ? (N + GSB_POINTS_THREADS - 1) / GSB_POINTS_THREADS : 0;
    const long long cap = mgrad ? (long long)GSB_RS_GRAD_PARTIAL_BLOCKS : 16LL * 148;
    if (blocks > cap) blocks = cap;
    const bool lens = model != GSB_LENS_PINHOLE;
    if (blocks > 0) {
        if (lens) {
            if (depth) launch_defocus_rs<true, true>(rolling != 0, mgrad != 0, (int)blocks, p);
            else launch_defocus_rs<false, true>(rolling != 0, mgrad != 0, (int)blocks, p);
        } else {
            if (depth) launch_defocus_rs<true, false>(rolling != 0, mgrad != 0, (int)blocks, p);
            else launch_defocus_rs<false, false>(rolling != 0, mgrad != 0, (int)blocks, p);
        }
    }
    if (mgrad) {
        struct FinishArgs {
            const float *partials;
            int blocks;
            float *g;
        } f{partials, (int)blocks, partials + (size_t)GSB_RS_GRAD_PARTIAL_BLOCKS * RS_GRAD_VALUES};
        simt_emu::launch([](const FinishArgs &a) { rolling_shutter_grad_finish_kernel(a.partials, a.blocks, a.g); }, 1,
                         RS_GRAD_FINISH_THREADS, f);
        grad_defocus[0] = f.g[0];  // the device-to-device copy of launch_backward_points_blur
        grad_defocus[1] = f.g[1];
    }
    return (int)blocks;
}
