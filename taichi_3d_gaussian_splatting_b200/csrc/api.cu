// api.cu -- extern "C" entry points of libgsb200.so (see include/gsb200.h).
#include <cstdarg>
#include <cstdio>
#include <cstring>

#include "common.cuh"

namespace gsb {

static thread_local char g_error[512] = "";

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_error, sizeof(g_error), fmt, ap);
    va_end(ap);
}

static inline int64_t align_up(int64_t v, int64_t a) { return (v + a - 1) / a * a; }

static int bit_width(uint64_t v) {
    int b = 0;
    while (v) {
        ++b;
        v >>= 1;
    }
    return b;
}

static int compute_layout(int64_t N, int32_t n_obj, int64_t key_capacity, int32_t H, int32_t W,
                          float far_plane, float depth_scale, uint32_t flags, GsbWorkspaceLayout *L) {
    if (!L) {
        set_error("workspace_layout: out is null");
        return GSB_EINVAL;
    }
    if (N < 0 || n_obj < 0 || key_capacity < 0 || H <= 0 || W <= 0) {
        set_error("workspace_layout: negative size (N=%lld n_obj=%d K_cap=%lld H=%d W=%d)", (long long)N,
                  n_obj, (long long)key_capacity, H, W);
        return GSB_EINVAL;
    }
    if (H % GSB_TILE_HEIGHT != 0 || W % GSB_TILE_WIDTH != 0) {  // GPCR:1193-1194
        set_error("camera size %dx%d must be a multiple of the 16x16 tile", W, H);
        return GSB_EINVAL;
    }
    if (N >= (1LL << 26) || key_capacity >= (1LL << 30)) {
        set_error("scene too large for the packed scan state (N < 2^26, key_capacity < 2^30)");
        return GSB_EUNSUPPORTED;
    }
    memset(L, 0, sizeof(*L));
    const int64_t T = (int64_t)(H / GSB_TILE_HEIGHT) * (W / GSB_TILE_WIDTH);
    L->tile_bits = bit_width((uint64_t)(T > 0 ? T - 1 : 0));
    const float mk = far_plane * depth_scale;  // f32 product, like the kernel's depth * scale
    int64_t max_key = mk >= 2147483648.0f ? 2147483647LL : (mk > 0.0f ? (int64_t)(int32_t)mk : 0);
    L->depth_bits = bit_width((uint64_t)max_key);
    if (L->depth_bits < 1) L->depth_bits = 1;
    if ((flags & GSB_FLAG_FORCE_KEY64) || L->tile_bits + L->depth_bits > 32) {
        L->key_bytes = 8;
        L->depth_bits = 32;  // exactly the reference's (tile << 32) + depth packing
    } else {
        L->key_bytes = 4;
    }
    L->radix_bits = sort_radix_bits(L->tile_bits + L->depth_bits);
    L->sort_passes = (L->tile_bits + L->depth_bits + L->radix_bits - 1) / L->radix_bits;
    if (L->sort_passes < 1) L->sort_passes = 1;
    L->key_capacity_padded = align_up(key_capacity > 0 ? key_capacity : 1, SORT_TILE);
    L->sort_blocks = (int32_t)(L->key_capacity_padded / SORT_TILE);
    L->scan_blocks = (int32_t)((N + SCAN_BLOCK_THREADS - 1) / SCAN_BLOCK_THREADS);

    int64_t off = 0;
    auto take = [&](int64_t bytes) {
        int64_t o = off;
        off = align_up(off + bytes, 256);
        return o;
    };
    L->counters = take(8 * sizeof(int64_t));
    L->tickets = take(16 * sizeof(uint32_t));
    L->scan_state = take((int64_t)(L->scan_blocks + 1) * 8);
    L->sort_hist = take(8 * 1024 * 4);
    L->sort_state = take((int64_t)L->sort_passes * L->sort_blocks * (1 << L->radix_bits) * 4);
    L->tile_start = take(T * 4);
    L->tile_end = take(T * 4);
    L->zero_bytes = off;
    L->poses = take((int64_t)(n_obj > 0 ? n_obj : 1) * sizeof(PoseBlock));
    L->point_id = take(N * 4);
    L->point_offset = take(N * 4);
    L->num_tiles = take(N * 4);
    L->records = take(N * GSB_RECORD_FLOATS * 4);
    L->point_in_camera = take(N * 3 * 4);
    L->keys_a = take(L->key_capacity_padded * L->key_bytes);
    L->keys_b = take(L->key_capacity_padded * L->key_bytes);
    L->vals_a = take(L->key_capacity_padded * 4);
    L->vals_b = take(L->key_capacity_padded * 4);
    L->keys_c = take(L->key_capacity_padded * L->key_bytes);
    L->vals_c = take(L->key_capacity_padded * 4);
    L->total_bytes = off;
    return GSB_OK;
}

int resolve_workspace(void *base, int64_t bytes, int64_t N, int32_t n_obj, int64_t key_capacity,
                      int32_t H, int32_t W, float far_plane, float depth_scale, uint32_t flags,
                      Workspace *ws) {
    int rc = compute_layout(N, n_obj, key_capacity, H, W, far_plane, depth_scale, flags, &ws->layout);
    if (rc != GSB_OK) return rc;
    const GsbWorkspaceLayout &L = ws->layout;
    if (!base || bytes < L.total_bytes) {
        set_error("workspace too small: have %lld bytes, need %lld", (long long)bytes, (long long)L.total_bytes);
        return GSB_EWORKSPACE;
    }
    if (reinterpret_cast<uintptr_t>(base) % 256 != 0) {
        set_error("workspace must be 256-byte aligned");
        return GSB_EINVAL;
    }
    char *b = static_cast<char *>(base);
    ws->counters = reinterpret_cast<long long *>(b + L.counters);
    ws->tickets = reinterpret_cast<unsigned int *>(b + L.tickets);
    ws->scan_state = reinterpret_cast<unsigned long long *>(b + L.scan_state);
    ws->sort_hist = reinterpret_cast<unsigned int *>(b + L.sort_hist);
    ws->sort_state = reinterpret_cast<unsigned int *>(b + L.sort_state);
    ws->tile_start = reinterpret_cast<int *>(b + L.tile_start);
    ws->tile_end = reinterpret_cast<int *>(b + L.tile_end);
    ws->poses = reinterpret_cast<PoseBlock *>(b + L.poses);
    ws->point_id = reinterpret_cast<int *>(b + L.point_id);
    ws->point_offset = reinterpret_cast<int *>(b + L.point_offset);
    ws->num_tiles = reinterpret_cast<int *>(b + L.num_tiles);
    ws->records = reinterpret_cast<float4 *>(b + L.records);
    ws->point_in_camera = reinterpret_cast<float *>(b + L.point_in_camera);
    ws->keys_a = b + L.keys_a;
    ws->keys_b = b + L.keys_b;
    ws->vals_a = reinterpret_cast<int *>(b + L.vals_a);
    ws->vals_b = reinterpret_cast<int *>(b + L.vals_b);
    ws->keys_c = b + L.keys_c;
    ws->vals_c = reinterpret_cast<int *>(b + L.vals_c);
    return GSB_OK;
}

static int check_forward_args(const GsbForwardArgs *a) {
    if (!a) {
        set_error("forward: args is null");
        return GSB_EINVAL;
    }
    if (a->num_points > 0 && (!a->pointcloud || !a->pointcloud_features || !a->point_invalid_mask ||
                              !a->point_object_id)) {
        set_error("forward: null scene pointer");
        return GSB_EINVAL;
    }
    if (a->num_points > 0 && (a->num_objects <= 0 || !a->q_pointcloud_camera || !a->t_pointcloud_camera)) {
        set_error("forward: need at least one object pose");
        return GSB_EINVAL;
    }
    if (!a->camera_intrinsics || !a->rasterized_image) {
        set_error("forward: null camera_intrinsics / rasterized_image");
        return GSB_EINVAL;
    }
    if (!a->rgb_only && (!a->rasterized_depth || !a->pixel_accumulated_alpha ||
                         !a->pixel_offset_of_last_effective_point || !a->pixel_valid_point_count)) {
        set_error("forward: aux outputs are required unless rgb_only");
        return GSB_EINVAL;
    }
    if (a->near_plane < 0.0f) {
        set_error("forward: near_plane must be >= 0 (depth keys are unsigned)");
        return GSB_EUNSUPPORTED;
    }
    if (reinterpret_cast<uintptr_t>(a->pointcloud_features) % 16 != 0) {
        set_error("forward: pointcloud_features must be 16-byte aligned");
        return GSB_EINVAL;
    }
    return GSB_OK;
}

static int resolve_fwd(const GsbForwardArgs *a, Workspace *ws) {
    int rc = check_forward_args(a);
    if (rc != GSB_OK) return rc;
    return resolve_workspace(a->workspace, a->workspace_bytes, a->num_points, a->num_objects,
                             a->key_capacity, a->camera_height, a->camera_width, a->far_plane,
                             a->depth_to_sort_key_scale, a->flags, ws);
}

}  // namespace gsb

using namespace gsb;

extern "C" {

int gsb200_version(void) { return GSB200_VERSION; }

const char *gsb200_last_error(void) { return g_error; }

void gsb200_abi_sizes(int64_t *out3) {
    out3[0] = (int64_t)sizeof(GsbWorkspaceLayout);
    out3[1] = (int64_t)sizeof(GsbForwardArgs);
    out3[2] = (int64_t)sizeof(GsbBackwardArgs);
}

void gsb200_abi_sizes_ext(int64_t *out, int32_t n) {
    const int64_t all[15] = {(int64_t)sizeof(GsbWorkspaceLayout), (int64_t)sizeof(GsbForwardArgs), (int64_t)sizeof(GsbBackwardArgs),
                             (int64_t)sizeof(GsbExpandArgs), (int64_t)sizeof(GsbTrainStepArgs), (int64_t)sizeof(GsbSupervisionArgs),
                             (int64_t)sizeof(GsbExtraFeatureArgs), (int64_t)sizeof(GsbFeatureTrainArgs),
                             (int64_t)sizeof(GsbPoseGradArgs), (int64_t)sizeof(GsbIntrinsicsGradArgs), (int64_t)sizeof(GsbLensArgs),
                             (int64_t)sizeof(GsbLensGradArgs), (int64_t)sizeof(GsbRollingShutterArgs),
                             (int64_t)sizeof(GsbRollingShutterGradArgs), (int64_t)sizeof(GsbAppearanceArgs)};
    for (int i = 0; i < n && i < 15; ++i) out[i] = all[i];
}

void gsb200_abi_sizes_mcmc(int64_t *out2) {
    out2[0] = (int64_t)sizeof(GsbMcmcRelocateArgs);
    out2[1] = (int64_t)sizeof(GsbMcmcStepArgs);
}

void gsb200_abi_sizes_filter3d(int64_t *out2) {
    out2[0] = (int64_t)sizeof(GsbFilter3dArgs);
    out2[1] = (int64_t)sizeof(GsbFilter3dViewsArgs);
}

int gsb200_workspace_layout(int64_t num_points, int32_t num_objects, int64_t key_capacity,
                            int32_t camera_height, int32_t camera_width, float far_plane,
                            float depth_to_sort_key_scale, uint32_t flags, GsbWorkspaceLayout *out) {
    return compute_layout(num_points, num_objects, key_capacity, camera_height, camera_width, far_plane,
                          depth_to_sort_key_scale, flags, out);
}

int gsb200_stage_preprocess(const GsbForwardArgs *a) {
    Workspace ws;
    int rc = resolve_fwd(a, &ws);
    if (rc != GSB_OK) return rc;
    return launch_preprocess(*a, ws, static_cast<cudaStream_t>(a->stream));
}

int gsb200_stage_sort(const GsbForwardArgs *a) {
    Workspace ws;
    int rc = resolve_fwd(a, &ws);
    if (rc != GSB_OK) return rc;
    return launch_sort(ws, a->key_capacity, static_cast<cudaStream_t>(a->stream));
}

int gsb200_stage_tile_ranges(const GsbForwardArgs *a) {
    Workspace ws;
    int rc = resolve_fwd(a, &ws);
    if (rc != GSB_OK) return rc;
    const int T = (a->camera_height / GSB_TILE_HEIGHT) * (a->camera_width / GSB_TILE_WIDTH);
    return launch_tile_ranges(ws, a->key_capacity, T, static_cast<cudaStream_t>(a->stream));
}

int gsb200_stage_blend(const GsbForwardArgs *a) {
    Workspace ws;
    int rc = resolve_fwd(a, &ws);
    if (rc != GSB_OK) return rc;
    return launch_blend_forward(*a, ws, static_cast<cudaStream_t>(a->stream));
}

int gsb200_forward(const GsbForwardArgs *a) { return gsb200_forward_ext(a, nullptr); }

// GsbLensArgs -> LensParams with the r^2 bound; GSB_EINVAL for an unknown model, a non-finite coefficient or a non-zero
// unused one.  *out_lens stays NULL for a NULL lens or GSB_LENS_PINHOLE (the default kernels).
static int check_lens(const char *what, const GsbLensArgs *lens, LensParams *params, const LensParams **out_lens) {
    *out_lens = nullptr;
    if (!lens) return GSB_OK;
    if (lens->model != GSB_LENS_PINHOLE && lens->model != GSB_LENS_OPENCV && lens->model != GSB_LENS_FISHEYE) {
        set_error("%s: unknown lens model %d", what, lens->model);
        return GSB_EINVAL;
    }
    const int used = lens->model == GSB_LENS_OPENCV ? 5 : lens->model == GSB_LENS_FISHEYE ? 4 : 0;
    for (int i = 0; i < 5; ++i) {
        const float k = lens->coefficients[i];
        if (!(k - k == 0.0f)) {
            set_error("%s: lens coefficient %d is not finite", what, i);
            return GSB_EINVAL;
        }
        if (i >= used && k != 0.0f) {
            set_error("%s: lens coefficient %d is not used by model %d and must be 0", what, i, lens->model);
            return GSB_EINVAL;
        }
    }
    if (lens->model == GSB_LENS_PINHOLE) return GSB_OK;
    params->model = lens->model;
    for (int i = 0; i < 5; ++i) params->k[i] = lens->coefficients[i];
    params->r2_max = (float)lens_r2_bound(lens->model, lens->coefficients);
    *out_lens = params;
    return GSB_OK;
}

int gsb200_forward_ext(const GsbForwardArgs *a, const GsbExtraFeatureArgs *ext) { return gsb200_forward_lens(a, ext, nullptr); }

int gsb200_forward_lens(const GsbForwardArgs *a, const GsbExtraFeatureArgs *ext, const GsbLensArgs *lens_args) {
    return gsb200_forward_rolling_shutter(a, ext, lens_args, nullptr);
}

// GsbRollingShutterArgs -> RsParams; GSB_EINVAL for a non-finite motion or a NULL or misaligned row_time.  *out_rs stays NULL
// for a NULL rs.
static int check_rs(const char *what, const GsbRollingShutterArgs *rs, RsParams *params, const RsParams **out_rs) {
    *out_rs = nullptr;
    if (!rs) return GSB_OK;
    for (int i = 0; i < 6; ++i) {
        const float m = rs->motion[i];
        if (!(m - m == 0.0f)) {
            set_error("%s: rolling-shutter motion %d is not finite", what, i);
            return GSB_EINVAL;
        }
    }
    if (!rs->row_time) {
        set_error("%s: null row_time pointer", what);
        return GSB_EINVAL;
    }
    if (reinterpret_cast<uintptr_t>(rs->row_time) % 4 != 0) {
        set_error("%s: row_time must be 4-byte aligned", what);
        return GSB_EINVAL;
    }
    for (int i = 0; i < 6; ++i) params->motion[i] = rs->motion[i];
    params->row_time = rs->row_time;
    *out_rs = params;
    return GSB_OK;
}

int64_t gsb200_rolling_shutter_grad_temp_bytes(void) {
    return (int64_t)GSB_RS_GRAD_PARTIAL_BLOCKS * 6 * (int64_t)sizeof(float);
}

int gsb200_forward_rolling_shutter(const GsbForwardArgs *a, const GsbExtraFeatureArgs *ext, const GsbLensArgs *lens_args,
                                   const GsbRollingShutterArgs *rs_args) {
    return gsb200_forward_filter3d(a, ext, lens_args, rs_args, nullptr);
}

// GsbFilter3dArgs -> the (N,) filter array; GSB_EINVAL for a NULL or not 4-byte aligned array.  *out stays NULL for a NULL
// filter.
static int check_filter3d(const char *what, const GsbFilter3dArgs *filter, const float **out) {
    *out = nullptr;
    if (!filter) return GSB_OK;
    if (!filter->filter3d || reinterpret_cast<uintptr_t>(filter->filter3d) % 4 != 0) {
        set_error("%s: filter3d is NULL or not 4-byte aligned", what);
        return GSB_EINVAL;
    }
    *out = filter->filter3d;
    return GSB_OK;
}

int gsb200_forward_filter3d(const GsbForwardArgs *a, const GsbExtraFeatureArgs *ext, const GsbLensArgs *lens_args,
                            const GsbRollingShutterArgs *rs_args, const GsbFilter3dArgs *filter) {
    const float *filter3d;
    int frc = check_filter3d("forward_filter3d", filter, &filter3d);
    if (frc != GSB_OK) return frc;
    LensParams lens_params;
    const LensParams *lens;
    int lrc = check_lens(rs_args ? "forward_rolling_shutter" : "forward_lens", lens_args, &lens_params, &lens);
    if (lrc != GSB_OK) return lrc;
    RsParams rs_params;
    const RsParams *rs;
    if ((lrc = check_rs("forward_rolling_shutter", rs_args, &rs_params, &rs)) != GSB_OK) return lrc;
    if (ext) {
        if (ext->channels < 1 || ext->channels > 16) {
            set_error("forward_ext: channels must be in 1..16 (got %d)", ext->channels);
            return GSB_EINVAL;
        }
        if (!ext->features || !ext->rasterized) {
            set_error("forward_ext: null features / rasterized pointer");
            return GSB_EINVAL;
        }
        if (a && a->rgb_only) {
            set_error("forward_ext: the feature map needs the full forward (rgb_only is set)");
            return GSB_EINVAL;
        }
    }
    Workspace ws;
    int rc = resolve_fwd(a, &ws);
    if (rc != GSB_OK) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(a->stream);
    if ((rc = launch_preprocess(*a, ws, st, lens, rs, filter3d)) != GSB_OK) return rc;
    if (a->host_counters && a->host_counters_event) {
        GSB_CUDA_CHECK(cudaMemcpyAsync(a->host_counters, ws.counters, 4 * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
        GSB_CUDA_CHECK(cudaEventRecord(static_cast<cudaEvent_t>(a->host_counters_event), st));
    }
    if ((rc = launch_sort(ws, a->key_capacity, st)) != GSB_OK) return rc;
    const int T = (a->camera_height / GSB_TILE_HEIGHT) * (a->camera_width / GSB_TILE_WIDTH);
    if ((rc = launch_tile_ranges(ws, a->key_capacity, T, st)) != GSB_OK) return rc;
    return launch_blend_forward(*a, ws, st, ext);
}

// grad_depth / depth: both NULL (no depth term), or both set; grad_alpha: NULL (no alpha term) or set; ext: NULL (no feature
// term) or set.  The auxiliary terms are checked in gsb200_backward_ext.
static int backward_impl(const GsbBackwardArgs *a, bool skip_on_overflow, const float *grad_depth = nullptr,
                         const float *depth = nullptr, const float *grad_alpha = nullptr,
                         const GsbExtraFeatureArgs *ext = nullptr, const GsbPoseGradArgs *pose = nullptr,
                         const GsbIntrinsicsGradArgs *intr = nullptr, const LensParams *lens = nullptr,
                         const GsbLensGradArgs *lens_grad = nullptr, const RsParams *rs = nullptr,
                         const GsbRollingShutterGradArgs *rs_grad = nullptr, const float *filter3d = nullptr) {
    if (!a) {
        set_error("backward: args is null");
        return GSB_EINVAL;
    }
    const bool compact = (a->flags & GSB_FLAG_COMPACT_GRADS) != 0;
    if (!a->grad_rasterized_image || !a->pixel_accumulated_alpha ||
        !a->pixel_offset_of_last_effective_point || !a->magnitude_grad_viewspace_on_image ||
        !a->camera_intrinsics ||
        (a->num_points > 0 && (!a->pointcloud || !a->pointcloud_features || !a->point_object_id || !a->t_pointcloud_camera)) ||
        (a->num_points > 0 && !compact && (!a->grad_pointcloud || !a->grad_pointcloud_features)) ||
        (a->num_points > 0 && compact && (!a->grad_sum_compact || !a->grad_color_compact))) {
        set_error("backward: null pointer argument");
        return GSB_EINVAL;
    }
    {
        const void *ctl[6] = {a->ctl_accumulated_num_in_camera, a->ctl_accumulated_num_pixels,
                              a->ctl_accumulated_view_space_position_gradients,
                              a->ctl_accumulated_view_space_position_gradients_avg, a->ctl_accumulated_position_gradients,
                              a->ctl_accumulated_position_gradients_norm};
        int set = 0;
        for (const void *c : ctl) set += c != nullptr;
        if (set != 0 && set != 6) {
            set_error("backward: the six controller accumulators must be all NULL or all set");
            return GSB_EINVAL;
        }
        if (set == 6 && (a->flags & GSB_FLAG_NO_HOOK_STATS)) {
            set_error("backward: the controller accumulators need the hook statistics (GSB_FLAG_NO_HOOK_STATS is set)");
            return GSB_EINVAL;
        }
    }
    if (compact && reinterpret_cast<uintptr_t>(a->grad_sum_compact) % 16 != 0) {
        set_error("backward: grad_sum_compact must be 16-byte aligned");
        return GSB_EINVAL;
    }
    if (a->accum_rows > 0 && !a->accum) {
        set_error("backward: accum is null");
        return GSB_EINVAL;
    }
    if (ext && reinterpret_cast<uintptr_t>(ext->grad_features) % 16 != 0) {
        set_error("backward_ext: grad_features must be 16-byte aligned");
        return GSB_EINVAL;
    }
    Workspace ws;
    int rc = resolve_workspace(a->workspace, a->workspace_bytes, a->num_points, a->num_objects,
                               a->key_capacity, a->camera_height, a->camera_width, a->far_plane,
                               a->depth_to_sort_key_scale, a->flags, &ws);
    if (rc != GSB_OK) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(a->stream);
    if (a->accum_rows > 0)
        GSB_CUDA_CHECK(cudaMemsetAsync(a->accum, 0, (size_t)a->accum_rows * GSB_ACCUM_FLOATS * 4, st));
    if (ext && a->num_points > 0)  // the blend adds into the rows it reaches; every other row stays zero
        GSB_CUDA_CHECK(cudaMemsetAsync(ext->grad_features, 0, (size_t)a->num_points * ext->channels * 4, st));
    if ((rc = launch_blend_backward(*a, ws, st, grad_depth, depth, grad_alpha, ext)) != GSB_OK) return rc;
    if (filter3d)
        return launch_backward_points_filter(*a, ws, st, skip_on_overflow ? ws.counters + CNT_OVERFLOW : nullptr,
                                             grad_depth != nullptr, lens, rs, filter3d);
    if (rs) return launch_backward_points_rs(*a, ws, st, grad_depth != nullptr, lens, *rs, rs_grad);
    if (lens && lens_grad) return launch_backward_points_lens_grad(*a, ws, st, grad_depth != nullptr, *lens, *lens_grad);
    if (lens) return launch_backward_points_lens(*a, ws, st, grad_depth != nullptr, *lens);
    if (intr) return launch_backward_points_calib(*a, ws, st, grad_depth != nullptr, pose, *intr);
    if (pose) return launch_backward_points_pose(*a, ws, st, grad_depth != nullptr, *pose);
    return launch_backward_points(*a, ws, st, skip_on_overflow ? ws.counters + CNT_OVERFLOW : nullptr, grad_depth != nullptr);
}

int gsb200_backward(const GsbBackwardArgs *a) { return backward_impl(a, false); }

int gsb200_backward_aux(const GsbBackwardArgs *a, const float *grad_rasterized_depth, const float *rasterized_depth,
                        const float *grad_pixel_accumulated_alpha) {
    return gsb200_backward_ext(a, grad_rasterized_depth, rasterized_depth, grad_pixel_accumulated_alpha, nullptr);
}

int gsb200_backward_ext(const GsbBackwardArgs *a, const float *grad_rasterized_depth, const float *rasterized_depth,
                        const float *grad_pixel_accumulated_alpha, const GsbExtraFeatureArgs *ext) {
    return gsb200_backward_pose(a, grad_rasterized_depth, rasterized_depth, grad_pixel_accumulated_alpha, ext, nullptr);
}

// gsb200_backward_calib's checks and dispatch; `lens` (gsb200_backward_lens, checked there) comes with neither pose nor
// intrinsics, `lens_grad` (gsb200_backward_lens_grad, checked there) only with `lens`, and `rs` / `rs_grad`
// (gsb200_backward_rolling_shutter, checked there) with neither pose, intrinsics nor lens_grad
static int backward_checked(const GsbBackwardArgs *a, const float *grad_rasterized_depth, const float *rasterized_depth,
                            const float *grad_pixel_accumulated_alpha, const GsbExtraFeatureArgs *ext, const GsbPoseGradArgs *pose,
                            const GsbIntrinsicsGradArgs *intr, const LensParams *lens, const GsbLensGradArgs *lens_grad = nullptr,
                            const RsParams *rs = nullptr, const GsbRollingShutterGradArgs *rs_grad = nullptr,
                            const float *filter3d = nullptr);

int gsb200_backward_filter3d(const GsbBackwardArgs *a, const float *grad_rasterized_depth, const float *rasterized_depth,
                             const float *grad_pixel_accumulated_alpha, const GsbExtraFeatureArgs *ext, const GsbLensArgs *lens_args,
                             const GsbRollingShutterArgs *rs_args, const GsbFilter3dArgs *filter) {
    if (!filter)
        return gsb200_backward_rolling_shutter(a, grad_rasterized_depth, rasterized_depth, grad_pixel_accumulated_alpha, ext,
                                               lens_args, rs_args, nullptr);
    const float *filter3d;
    int rc = check_filter3d("backward_filter3d", filter, &filter3d);
    if (rc != GSB_OK) return rc;
    LensParams lens_params;
    const LensParams *lens;
    if ((rc = check_lens("backward_filter3d", lens_args, &lens_params, &lens)) != GSB_OK) return rc;
    RsParams rs_params;
    const RsParams *rs;
    if ((rc = check_rs("backward_filter3d", rs_args, &rs_params, &rs)) != GSB_OK) return rc;
    if (a != nullptr && (a->flags & GSB_FLAG_COMPACT_GRADS)) {
        set_error("backward_filter3d: the 3D filter is not implemented for the compact rows of the view-parallel exchange "
                  "(GSB_FLAG_COMPACT_GRADS)");
        return GSB_EUNSUPPORTED;
    }
    return backward_checked(a, grad_rasterized_depth, rasterized_depth, grad_pixel_accumulated_alpha, ext, nullptr, nullptr, lens,
                            nullptr, rs, nullptr, filter3d);
}

int gsb200_backward_rolling_shutter(const GsbBackwardArgs *a, const float *grad_rasterized_depth, const float *rasterized_depth,
                                    const float *grad_pixel_accumulated_alpha, const GsbExtraFeatureArgs *ext,
                                    const GsbLensArgs *lens_args, const GsbRollingShutterArgs *rs_args,
                                    const GsbRollingShutterGradArgs *rs_grad) {
    if (!rs_args && rs_grad) {
        set_error("backward_rolling_shutter: the motion gradient needs a rolling shutter (rs is NULL)");
        return GSB_EINVAL;
    }
    if (!rs_args) return gsb200_backward_lens(a, grad_rasterized_depth, rasterized_depth, grad_pixel_accumulated_alpha, ext, lens_args);
    LensParams lens_params;
    const LensParams *lens;
    int rc = check_lens("backward_rolling_shutter", lens_args, &lens_params, &lens);
    if (rc != GSB_OK) return rc;
    RsParams rs_params;
    const RsParams *rs;
    if ((rc = check_rs("backward_rolling_shutter", rs_args, &rs_params, &rs)) != GSB_OK) return rc;
    if (rs_grad) {
        if (!rs_grad->grad_motion || !rs_grad->temp) {
            set_error("backward_rolling_shutter: null grad_motion / temp pointer");
            return GSB_EINVAL;
        }
        if (reinterpret_cast<uintptr_t>(rs_grad->grad_motion) % 4 != 0) {
            set_error("backward_rolling_shutter: grad_motion must be 4-byte aligned");
            return GSB_EINVAL;
        }
        if (reinterpret_cast<uintptr_t>(rs_grad->temp) % 16 != 0) {
            set_error("backward_rolling_shutter: the rolling-shutter temp must be 16-byte aligned");
            return GSB_EINVAL;
        }
    }
    if (a != nullptr && (a->flags & GSB_FLAG_COMPACT_GRADS)) {
        set_error("backward_rolling_shutter: the rolling shutter is not implemented for the compact rows of the view-parallel "
                  "exchange (GSB_FLAG_COMPACT_GRADS)");
        return GSB_EUNSUPPORTED;
    }
    return backward_checked(a, grad_rasterized_depth, rasterized_depth, grad_pixel_accumulated_alpha, ext, nullptr, nullptr, lens,
                            nullptr, rs, rs_grad);
}

int gsb200_backward_lens(const GsbBackwardArgs *a, const float *grad_rasterized_depth, const float *rasterized_depth,
                         const float *grad_pixel_accumulated_alpha, const GsbExtraFeatureArgs *ext, const GsbLensArgs *lens_args) {
    LensParams lens_params;
    const LensParams *lens;
    int rc = check_lens("backward_lens", lens_args, &lens_params, &lens);
    if (rc != GSB_OK) return rc;
    if (!lens) return gsb200_backward_ext(a, grad_rasterized_depth, rasterized_depth, grad_pixel_accumulated_alpha, ext);
    if (a != nullptr && (a->flags & GSB_FLAG_COMPACT_GRADS)) {
        set_error("backward_lens: the lens gradient is not implemented for the compact rows of the view-parallel exchange "
                  "(GSB_FLAG_COMPACT_GRADS)");
        return GSB_EUNSUPPORTED;
    }
    return backward_checked(a, grad_rasterized_depth, rasterized_depth, grad_pixel_accumulated_alpha, ext, nullptr, nullptr, lens);
}

int64_t gsb200_lens_grad_temp_bytes(void) {
    return (int64_t)GSB_LENS_GRAD_PARTIAL_BLOCKS * 5 * (int64_t)sizeof(float);
}

int gsb200_backward_lens_grad(const GsbBackwardArgs *a, const float *grad_rasterized_depth, const float *rasterized_depth,
                              const float *grad_pixel_accumulated_alpha, const GsbExtraFeatureArgs *ext,
                              const GsbLensArgs *lens_args, const GsbLensGradArgs *lens_grad) {
    if (!lens_grad) return gsb200_backward_lens(a, grad_rasterized_depth, rasterized_depth, grad_pixel_accumulated_alpha, ext, lens_args);
    LensParams lens_params;
    const LensParams *lens;
    int rc = check_lens("backward_lens_grad", lens_args, &lens_params, &lens);
    if (rc != GSB_OK) return rc;
    if (!lens) {
        set_error("backward_lens_grad: the coefficient gradient needs an opencv or fisheye lens (got %s)",
                  lens_args ? "GSB_LENS_PINHOLE" : "NULL");
        return GSB_EINVAL;
    }
    if (!lens_grad->grad_coefficients || !lens_grad->temp) {
        set_error("backward_lens_grad: null grad_coefficients / temp pointer");
        return GSB_EINVAL;
    }
    if (reinterpret_cast<uintptr_t>(lens_grad->grad_coefficients) % 4 != 0) {
        set_error("backward_lens_grad: grad_coefficients must be 4-byte aligned");
        return GSB_EINVAL;
    }
    if (reinterpret_cast<uintptr_t>(lens_grad->temp) % 16 != 0) {
        set_error("backward_lens_grad: the lens temp must be 16-byte aligned");
        return GSB_EINVAL;
    }
    if (a != nullptr && (a->flags & GSB_FLAG_COMPACT_GRADS)) {
        set_error("backward_lens_grad: the lens gradient is not implemented for the compact rows of the view-parallel exchange "
                  "(GSB_FLAG_COMPACT_GRADS)");
        return GSB_EUNSUPPORTED;
    }
    return backward_checked(a, grad_rasterized_depth, rasterized_depth, grad_pixel_accumulated_alpha, ext, nullptr, nullptr, lens,
                            lens_grad);
}

int64_t gsb200_pose_grad_temp_bytes(int32_t num_objects) {
    return num_objects < 1 ? 0 : (int64_t)GSB_POSE_PARTIAL_BLOCKS * num_objects * 12 * (int64_t)sizeof(float);
}

int gsb200_backward_pose(const GsbBackwardArgs *a, const float *grad_rasterized_depth, const float *rasterized_depth,
                         const float *grad_pixel_accumulated_alpha, const GsbExtraFeatureArgs *ext, const GsbPoseGradArgs *pose) {
    return gsb200_backward_calib(a, grad_rasterized_depth, rasterized_depth, grad_pixel_accumulated_alpha, ext, pose, nullptr);
}

int64_t gsb200_intrinsics_grad_temp_bytes(void) {
    return (int64_t)GSB_INTRINSICS_PARTIAL_BLOCKS * 6 * (int64_t)sizeof(float);
}

int gsb200_backward_calib(const GsbBackwardArgs *a, const float *grad_rasterized_depth, const float *rasterized_depth,
                          const float *grad_pixel_accumulated_alpha, const GsbExtraFeatureArgs *ext, const GsbPoseGradArgs *pose,
                          const GsbIntrinsicsGradArgs *intr) {
    return backward_checked(a, grad_rasterized_depth, rasterized_depth, grad_pixel_accumulated_alpha, ext, pose, intr, nullptr);
}

static int backward_checked(const GsbBackwardArgs *a, const float *grad_rasterized_depth, const float *rasterized_depth,
                            const float *grad_pixel_accumulated_alpha, const GsbExtraFeatureArgs *ext, const GsbPoseGradArgs *pose,
                            const GsbIntrinsicsGradArgs *intr, const LensParams *lens, const GsbLensGradArgs *lens_grad,
                            const RsParams *rs, const GsbRollingShutterGradArgs *rs_grad, const float *filter3d) {
    if (intr) {
        if (!intr->grad_camera_intrinsics || !intr->temp) {
            set_error("backward_calib: null grad_camera_intrinsics / temp pointer");
            return GSB_EINVAL;
        }
        if (reinterpret_cast<uintptr_t>(intr->temp) % 16 != 0) {
            set_error("backward_calib: the intrinsics temp must be 16-byte aligned");
            return GSB_EINVAL;
        }
        if (a != nullptr && (a->flags & GSB_FLAG_COMPACT_GRADS)) {
            set_error("backward_calib: the intrinsics gradient is not implemented for the compact rows of the view-parallel "
                      "exchange (GSB_FLAG_COMPACT_GRADS)");
            return GSB_EUNSUPPORTED;
        }
    }
    if (pose) {
        if (!pose->q_pointcloud_camera || !pose->grad_q_pointcloud_camera || !pose->grad_t_pointcloud_camera || !pose->temp) {
            set_error("backward_pose: null q_pointcloud_camera / grad_q_pointcloud_camera / grad_t_pointcloud_camera / temp "
                      "pointer");
            return GSB_EINVAL;
        }
        if (reinterpret_cast<uintptr_t>(pose->temp) % 16 != 0) {
            set_error("backward_pose: temp must be 16-byte aligned");
            return GSB_EINVAL;
        }
        if (a != nullptr && a->num_objects < 1) {
            set_error("backward_pose: the pose gradient needs num_objects >= 1 (got %d)", a->num_objects);
            return GSB_EINVAL;
        }
        if (a != nullptr && a->num_objects > GSB_POSE_MAX_OBJECTS) {
            set_error("backward_pose: at most GSB_POSE_MAX_OBJECTS = %d objects (got %d)", GSB_POSE_MAX_OBJECTS, a->num_objects);
            return GSB_EUNSUPPORTED;
        }
        if (a != nullptr && (a->flags & GSB_FLAG_COMPACT_GRADS)) {
            set_error("backward_pose: the pose gradient is not implemented for the compact rows of the view-parallel exchange "
                      "(GSB_FLAG_COMPACT_GRADS)");
            return GSB_EUNSUPPORTED;
        }
    }
    if ((grad_rasterized_depth == nullptr) != (rasterized_depth == nullptr)) {
        set_error("backward_aux: grad_rasterized_depth and rasterized_depth must be both NULL or both set");
        return GSB_EINVAL;
    }
    if (ext) {
        if (ext->channels < 1 || ext->channels > 16) {
            set_error("backward_ext: channels must be in 1..16 (got %d)", ext->channels);
            return GSB_EINVAL;
        }
        if (!ext->features || !ext->grad_rasterized || !ext->grad_features) {
            set_error("backward_ext: null features / grad_rasterized / grad_features pointer");
            return GSB_EINVAL;
        }
        if (a != nullptr && (a->flags & GSB_FLAG_COMPACT_GRADS)) {
            set_error("backward_ext: the feature gradient is not carried by the compact rows of the view-parallel exchange "
                      "(GSB_FLAG_COMPACT_GRADS)");
            return GSB_EUNSUPPORTED;
        }
    }
    const bool aux = grad_rasterized_depth != nullptr || grad_pixel_accumulated_alpha != nullptr || ext != nullptr;
    if (aux && a != nullptr && !(a->flags & GSB_FLAG_BACKWARD_TRANSPOSED)) {
        set_error("backward_aux: the depth, alpha and feature gradients need the transposed backward kernel "
                  "(GSB_FLAG_BACKWARD_TRANSPOSED); the butterfly kernel does not implement them");
        return GSB_EUNSUPPORTED;
    }
    return backward_impl(a, false, grad_rasterized_depth, rasterized_depth, grad_pixel_accumulated_alpha, ext, pose, intr, lens,
                         lens_grad, rs, rs_grad, filter3d);
}

int gsb200_backward_with_depth(const GsbBackwardArgs *a, const float *grad_rasterized_depth, const float *rasterized_depth) {
    return gsb200_backward_aux(a, grad_rasterized_depth, rasterized_depth, nullptr);
}

int gsb200_image_loss(const float *rasterized_image, const float *ground_truth_image, int32_t camera_height,
                      int32_t camera_width, float lambda_value, float upstream_grad, float *loss_out3,
                      float *grad_rasterized_image, void *temp, int64_t temp_bytes, void *stream);

static bool weight_ok(float w) { return w >= 0.0f && w <= 3.402823466e38f; }  // false for NaN, inf and negatives

int gsb200_train_step(const GsbTrainStepArgs *t) { return gsb200_train_step_aux(t, nullptr); }

int gsb200_train_step_aux(const GsbTrainStepArgs *t, const GsbSupervisionArgs *s) { return gsb200_train_step_ext(t, s, nullptr); }

static bool aligned16(const void *p) { return reinterpret_cast<uintptr_t>(p) % 16 == 0; }

// The feature term's own rules (gsb200_train_step_ext); the frame's were checked before.
static int check_feature_train_args(const GsbFeatureTrainArgs &x, const GsbBackwardArgs &b, int H, int W) {
    const GsbExtraFeatureArgs &e = x.features;
    if (e.channels < 1 || e.channels > 16) {
        set_error("train_step_ext: channels must be in 1..16 (got %d)", e.channels);
        return GSB_EINVAL;
    }
    if (x.loss_kind != GSB_FEATURE_LOSS_CROSS_ENTROPY && x.loss_kind != GSB_FEATURE_LOSS_L2) {
        set_error("train_step_ext: unknown feature loss kind %d", x.loss_kind);
        return GSB_EINVAL;
    }
    const bool ce = x.loss_kind == GSB_FEATURE_LOSS_CROSS_ENTROPY;
    if (ce && e.channels < 2) {
        set_error("train_step_ext: the cross-entropy feature loss needs C >= 2 channels (got %d)", e.channels);
        return GSB_EINVAL;
    }
    if (!(x.weight > 0.0f && x.weight <= 3.402823466e38f)) {
        set_error("train_step_ext: the feature loss weight must be finite and > 0 (got %g)", (double)x.weight);
        return GSB_EINVAL;
    }
    if ((ce ? (const void *)x.labels : (const void *)x.target) == nullptr) {
        set_error("train_step_ext: the %s feature loss needs its target (%s)", ce ? "cross-entropy" : "l2",
                  ce ? "labels" : "target");
        return GSB_EINVAL;
    }
    if (!e.features || !e.rasterized || !e.grad_rasterized || !e.grad_features || !x.exp_avg || !x.exp_avg_sq ||
        !x.loss_out2) {
        set_error("train_step_ext: null features / rasterized / grad_rasterized / grad_features / exp_avg / exp_avg_sq / "
                  "loss_out2 pointer");
        return GSB_EINVAL;
    }
    if (!x.temp || !aligned16(x.temp) || x.temp_bytes < gsb200_feature_loss_temp_bytes(H, W)) {
        set_error("train_step_ext: feature temp null, not 16-byte aligned or smaller than gsb200_feature_loss_temp_bytes(H, W) "
                  "(temp_bytes=%lld)", (long long)x.temp_bytes);
        return GSB_EINVAL;
    }
    if (!aligned16(e.features) || !aligned16(e.grad_features) || !aligned16(x.exp_avg) || !aligned16(x.exp_avg_sq)) {
        set_error("train_step_ext: features, grad_features, exp_avg and exp_avg_sq must be 16-byte aligned");
        return GSB_EINVAL;
    }
    if (!(b.flags & GSB_FLAG_BACKWARD_TRANSPOSED)) {
        set_error("train_step_ext: the feature gradient needs the transposed backward kernel (GSB_FLAG_BACKWARD_TRANSPOSED)");
        return GSB_EUNSUPPORTED;
    }
    return GSB_OK;
}

// The appearance grid's own rules (gsb200_train_step_appearance); the frame's were checked before.
static int check_appearance_args(const GsbAppearanceArgs &a, int H, int W) {
    if (a.grid_x < 1 || a.grid_x > GSB_BILATERAL_GRID_MAX_XY || a.grid_y < 1 || a.grid_y > GSB_BILATERAL_GRID_MAX_XY ||
        a.grid_z < 1 || a.grid_z > GSB_BILATERAL_GRID_MAX_Z) {
        set_error("train_step_appearance: the grid must have 1 <= Gx, Gy <= %d and 1 <= Gz <= %d nodes (got %dx%dx%d)",
                  GSB_BILATERAL_GRID_MAX_XY, GSB_BILATERAL_GRID_MAX_Z, a.grid_x, a.grid_y, a.grid_z);
        return GSB_EINVAL;
    }
    if (!weight_ok(a.tv_weight) || !(a.learning_rate >= 0.0 && a.learning_rate <= 1.7976931348623157e308)) {
        set_error("train_step_appearance: the TV weight and the learning rate must be finite and >= 0 (got %g, %g)",
                  (double)a.tv_weight, a.learning_rate);
        return GSB_EINVAL;
    }
    if (a.step < 1) {
        set_error("train_step_appearance: the grid's step must be >= 1 (got %d)", a.step);
        return GSB_EINVAL;
    }
    if (!a.grid || !a.grad_grid || !a.exp_avg || !a.exp_avg_sq || !a.image || !a.loss_out1 || !aligned16(a.grid) ||
        !aligned16(a.grad_grid) || !aligned16(a.exp_avg) || !aligned16(a.exp_avg_sq) || !aligned16(a.image)) {
        set_error("train_step_appearance: grid, grad_grid, exp_avg, exp_avg_sq and image must be 16-byte aligned, "
                  "loss_out1 not NULL");
        return GSB_EINVAL;
    }
    if (!a.temp || !aligned16(a.temp) ||
        a.temp_bytes < gsb200_bilateral_grid_temp_bytes(H, W, a.grid_x, a.grid_y, a.grid_z)) {
        set_error("train_step_appearance: temp null, not 16-byte aligned or smaller than gsb200_bilateral_grid_temp_bytes "
                  "(temp_bytes=%lld)", (long long)a.temp_bytes);
        return GSB_EINVAL;
    }
    return GSB_OK;
}

int gsb200_train_step_ext(const GsbTrainStepArgs *t, const GsbSupervisionArgs *s, const GsbFeatureTrainArgs *x) {
    return gsb200_train_step_appearance(t, s, x, nullptr);
}

int gsb200_train_step_appearance(const GsbTrainStepArgs *t, const GsbSupervisionArgs *s, const GsbFeatureTrainArgs *x,
                                 const GsbAppearanceArgs *app) {
    return gsb200_train_step_mcmc(t, s, x, app, nullptr);
}

// The rules of the regulariser and of the noise (gsb200_mcmc_regulariser, gsb200_mcmc_noise, gsb200_train_step_mcmc).
static int check_mcmc_regulariser(const char *what, int64_t N, int64_t num_valid, float lambda_opacity, float lambda_scale,
                                  const float *terms_out, const void *temp) {
    if (N < 0 || num_valid < 0 || num_valid > N) {
        set_error("%s: num_valid must be in [0, num_points] (got %lld of %lld)", what, (long long)num_valid, (long long)N);
        return GSB_EINVAL;
    }
    if (!weight_ok(lambda_opacity) || !weight_ok(lambda_scale)) {
        set_error("%s: the opacity and scale weights must be finite and >= 0 (got %g, %g)", what, (double)lambda_opacity,
                  (double)lambda_scale);
        return GSB_EINVAL;
    }
    if (!terms_out || !temp || !aligned16(temp)) {
        set_error("%s: terms_out2 NULL, or temp NULL or not 16-byte aligned", what);
        return GSB_EINVAL;
    }
    return GSB_OK;
}

static int check_mcmc_noise(const char *what, int64_t N, float noise_scale, float gate_k, float min_opacity, int64_t step) {
    if (N < 0 || step < 0) {
        set_error("%s: num_points and the noise step must be >= 0 (got %lld, %lld)", what, (long long)N, (long long)step);
        return GSB_EINVAL;
    }
    if (!weight_ok(noise_scale) || !weight_ok(gate_k) || !weight_ok(min_opacity)) {
        set_error("%s: noise_scale, gate_k and min_opacity must be finite and >= 0 (got %g, %g, %g)", what, (double)noise_scale,
                  (double)gate_k, (double)min_opacity);
        return GSB_EINVAL;
    }
    return GSB_OK;
}

int gsb200_mcmc_regulariser(const float *features, const int8_t *invalid_mask, float *grad_features, int64_t N,
                            int64_t num_valid, float lambda_opacity, float lambda_scale, float *terms_out2, void *temp,
                            void *stream) {
    int rc = check_mcmc_regulariser("mcmc_regulariser", N, num_valid, lambda_opacity, lambda_scale, terms_out2, temp);
    if (rc != GSB_OK) return rc;
    if (!features || !invalid_mask || !grad_features || !aligned16(features) || !aligned16(grad_features)) {
        set_error("mcmc_regulariser: NULL pointer, or features / grad_features not 16-byte aligned");
        return GSB_EINVAL;
    }
    return launch_mcmc_regulariser(features, invalid_mask, grad_features, N, num_valid, lambda_opacity, lambda_scale, terms_out2,
                                   temp, nullptr, static_cast<cudaStream_t>(stream));
}

int gsb200_mcmc_noise(float *pointcloud, const float *features, const int8_t *invalid_mask, int64_t N, float noise_scale,
                      float gate_k, float min_opacity, uint64_t seed, int64_t step, void *stream) {
    int rc = check_mcmc_noise("mcmc_noise", N, noise_scale, gate_k, min_opacity, step);
    if (rc != GSB_OK) return rc;
    if (!pointcloud || !features || !invalid_mask || reinterpret_cast<uintptr_t>(pointcloud) % 4 || !aligned16(features)) {
        set_error("mcmc_noise: NULL pointer, pointcloud not 4-byte aligned or features not 16-byte aligned");
        return GSB_EINVAL;
    }
    return launch_mcmc_noise(pointcloud, features, invalid_mask, N, noise_scale, gate_k, min_opacity, seed, step, nullptr,
                             static_cast<cudaStream_t>(stream));
}

int gsb200_train_step_mcmc(const GsbTrainStepArgs *t, const GsbSupervisionArgs *s, const GsbFeatureTrainArgs *x,
                           const GsbAppearanceArgs *app, const GsbMcmcStepArgs *mc) {
    return gsb200_train_step_filter3d(t, s, x, app, mc, nullptr);
}

int gsb200_train_step_filter3d(const GsbTrainStepArgs *t, const GsbSupervisionArgs *s, const GsbFeatureTrainArgs *x,
                               const GsbAppearanceArgs *app, const GsbMcmcStepArgs *mc, const GsbFilter3dArgs *filter) {
    return gsb200_train_step_robust(t, s, x, app, mc, filter, nullptr);
}

// The loss weights' own rules (gsb200_train_step_robust, gsb200_robust_image_loss).
static int check_robust_args(const char *what, const GsbRobustLossArgs &r, int H, int W) {
    if (r.robust != 0 && r.robust != 1) {
        set_error("%s: robust must be 0 or 1 (got %d)", what, r.robust);
        return GSB_EINVAL;
    }
    if (r.robust && (!(r.inlier_quantile > 0.0f && r.inlier_quantile <= 1.0f) ||
                     !(r.box_threshold >= 0.0f && r.box_threshold <= 1.0f) ||
                     !(r.patch_threshold >= 0.0f && r.patch_threshold <= 1.0f))) {
        set_error("%s: the inlier quantile must be in (0, 1] and the thresholds in [0, 1] (got %g, %g, %g)", what,
                  (double)r.inlier_quantile, (double)r.box_threshold, (double)r.patch_threshold);
        return GSB_EINVAL;
    }
    if (H < 16 || W < 16 || H % 16 || W % 16) {
        set_error("%s: the loss weights need H and W to be multiples of 16 (got %dx%d)", what, H, W);
        return GSB_EINVAL;
    }
    const auto aligned4 = [](const void *p) { return reinterpret_cast<uintptr_t>(p) % 4 == 0; };
    if (!r.weight_out || !r.composite || !r.stats_out2 || !aligned4(r.static_weight) || !aligned4(r.weight_out) ||
        !aligned4(r.composite)) {
        set_error("%s: NULL weight_out, composite or stats_out2, or a static weight, weight_out or composite that is not "
                  "4-byte aligned", what);
        return GSB_EINVAL;
    }
    if (!r.temp || !aligned16(r.temp) || r.temp_bytes < gsb200_robust_temp_bytes(H, W)) {
        set_error("%s: temp null, not 16-byte aligned or smaller than gsb200_robust_temp_bytes(H, W) (temp_bytes=%lld)", what,
                  (long long)r.temp_bytes);
        return GSB_EINVAL;
    }
    return GSB_OK;
}

int gsb200_robust_image_loss(const float *rasterized_image, const float *ground_truth_image, int32_t camera_height,
                             int32_t camera_width, float lambda_value, const GsbRobustLossArgs *robust, float *loss_out3,
                             float *grad_rasterized_image, void *temp, int64_t temp_bytes, void *stream) {
    if (!robust || !rasterized_image || !ground_truth_image || !grad_rasterized_image) {
        set_error("robust_image_loss: NULL robust, image, ground truth or gradient");
        return GSB_EINVAL;
    }
    int rc = check_robust_args("robust_image_loss", *robust, camera_height, camera_width);
    if (rc != GSB_OK) return rc;
    if (!loss_out3 || !temp || temp_bytes < gsb200_image_loss_temp_bytes(camera_height, camera_width) || !aligned16(temp)) {
        set_error("robust_image_loss: loss_out3 NULL, or the image loss's temp null, not 16-byte aligned or too small "
                  "(temp_bytes=%lld)", (long long)temp_bytes);
        return GSB_EINVAL;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if ((rc = launch_robust_pre(*robust, rasterized_image, ground_truth_image, camera_height, camera_width, st)) != GSB_OK)
        return rc;
    if ((rc = gsb200_image_loss(robust->composite, ground_truth_image, camera_height, camera_width, lambda_value, 1.0f,
                                loss_out3, grad_rasterized_image, temp, temp_bytes, stream)) != GSB_OK)
        return rc;
    return launch_robust_post(*robust, rasterized_image, camera_height, camera_width, grad_rasterized_image, st);
}

void gsb200_abi_sizes_robust(int64_t *out1) { out1[0] = (int64_t)sizeof(GsbRobustLossArgs); }

int gsb200_train_step_robust(const GsbTrainStepArgs *t, const GsbSupervisionArgs *s, const GsbFeatureTrainArgs *x,
                             const GsbAppearanceArgs *app, const GsbMcmcStepArgs *mc, const GsbFilter3dArgs *filter,
                             const GsbRobustLossArgs *robust) {
    const float *filter3d;
    int frc = check_filter3d("train_step_filter3d", filter, &filter3d);
    if (frc != GSB_OK) return frc;
    if (!t || !t->ground_truth_image || !t->loss_out3 || !t->loss_temp || !t->feature_exp_avg || !t->feature_exp_avg_sq ||
        !t->position_exp_avg || !t->position_exp_avg_sq || t->step < 1) {
        set_error("train_step: null pointer argument or step < 1");
        return GSB_EINVAL;
    }
    const GsbForwardArgs &f = t->forward;
    const GsbBackwardArgs &b = t->backward;
    if (x && (b.flags & GSB_FLAG_COMPACT_GRADS)) {
        set_error("train_step_ext: the feature gradient is not carried by the compact rows of the view-parallel exchange "
                  "(GSB_FLAG_COMPACT_GRADS)");
        return GSB_EUNSUPPORTED;
    }
    if (f.rgb_only || f.num_points != b.num_points || f.workspace != b.workspace || f.camera_height != b.camera_height ||
        f.camera_width != b.camera_width || f.stream != b.stream || b.accum_rows < f.num_points ||
        (b.flags & GSB_FLAG_COMPACT_GRADS) || !b.grad_rasterized_image || !b.grad_pointcloud || !b.grad_pointcloud_features ||
        b.pointcloud != f.pointcloud || b.pointcloud_features != f.pointcloud_features) {
        set_error("train_step: forward / backward blocks do not describe one frame (or rgb_only / compact gradients set)");
        return GSB_EINVAL;
    }
    bool depth_on = false, alpha_on = false;
    if (s) {
        if (!weight_ok(s->depth_weight) || !weight_ok(s->mask_weight)) {
            set_error("train_step_aux: the depth and mask weights must be finite and >= 0 (got %g, %g)", (double)s->depth_weight,
                      (double)s->mask_weight);
            return GSB_EINVAL;
        }
        depth_on = s->depth_weight > 0.0f;
        const bool mask_on = s->mask_weight > 0.0f;
        if (depth_on && (!s->depth_target || !s->grad_depth)) {
            set_error("train_step_aux: a depth weight > 0 needs depth_target and grad_depth");
            return GSB_EINVAL;
        }
        if (mask_on && !s->mask_target) {
            set_error("train_step_aux: a mask weight > 0 needs mask_target");
            return GSB_EINVAL;
        }
        alpha_on = mask_on || s->background != nullptr;
        if (alpha_on && !s->grad_pixel_accumulated_alpha) {
            set_error("train_step_aux: the mask term and the background need grad_pixel_accumulated_alpha");
            return GSB_EINVAL;
        }
        if (depth_on || alpha_on) {
            if (!s->loss_out3 || !s->temp || reinterpret_cast<uintptr_t>(s->temp) % 16 ||
                s->temp_bytes < gsb200_supervision_temp_bytes(f.camera_height, f.camera_width)) {
                set_error("train_step_aux: loss_out3 missing, or temp null, not 16-byte aligned or smaller than "
                          "gsb200_supervision_temp_bytes(H, W) (temp_bytes=%lld)", (long long)s->temp_bytes);
                return GSB_EINVAL;
            }
            if (!(b.flags & GSB_FLAG_BACKWARD_TRANSPOSED)) {
                set_error("train_step_aux: the depth and alpha gradients need the transposed backward kernel "
                          "(GSB_FLAG_BACKWARD_TRANSPOSED)");
                return GSB_EUNSUPPORTED;
            }
            if (!f.rasterized_depth || !f.pixel_accumulated_alpha) {
                set_error("train_step_aux: the supervision terms need the forward's depth and accumulated alpha outputs");
                return GSB_EINVAL;
            }
        }
    }
    const bool supervised = depth_on || alpha_on;
    const int H = f.camera_height, W = f.camera_width;
    int rc;
    if (x && (rc = check_feature_train_args(*x, b, H, W)) != GSB_OK) return rc;
    if (app && (rc = check_appearance_args(*app, H, W)) != GSB_OK) return rc;
    if (mc) {
        if ((rc = check_mcmc_regulariser("train_step_mcmc", f.num_points, mc->num_valid, mc->lambda_opacity, mc->lambda_scale,
                                         mc->terms_out2, mc->temp)) != GSB_OK)
            return rc;
        if ((rc = check_mcmc_noise("train_step_mcmc", f.num_points, mc->noise_scale, mc->gate_k, mc->min_opacity,
                                   mc->step)) != GSB_OK)
            return rc;
        if (!f.point_invalid_mask || !aligned16(f.pointcloud_features) || !aligned16(b.grad_pointcloud_features)) {
            set_error("train_step_mcmc: NULL invalid mask, or features / grad_features not 16-byte aligned");
            return GSB_EINVAL;
        }
    }
    if (robust) {
        if ((rc = check_robust_args("train_step_robust", *robust, H, W)) != GSB_OK) return rc;
        // the image loss runs between the robust pre- and post-passes: its rules are checked before either is launched
        if (t->loss_temp_bytes < gsb200_image_loss_temp_bytes(H, W) || !aligned16(t->loss_temp)) {
            set_error("train_step_robust: the image loss's temp is not 16-byte aligned or smaller than "
                      "gsb200_image_loss_temp_bytes(H, W) (loss_temp_bytes=%lld)", (long long)t->loss_temp_bytes);
            return GSB_EINVAL;
        }
    }
    const GsbExtraFeatureArgs *ext = x ? &x->features : nullptr;
    cudaStream_t st = static_cast<cudaStream_t>(f.stream);
    if ((rc = gsb200_forward_filter3d(&f, ext, nullptr, nullptr, filter)) != GSB_OK) return rc;
    const float *loss_image = f.rasterized_image, *loss_gt = t->ground_truth_image;
    if (supervised && (rc = launch_supervision_pre(*s, f.rasterized_image, t->ground_truth_image, f.pixel_accumulated_alpha,
                                                   f.rasterized_depth, H, W, st, &loss_image, &loss_gt)) != GSB_OK)
        return rc;
    const float *sliced_image = loss_image;  // I'' (the image loss's input)
    if (app) {
        if ((rc = launch_bilateral_grid_forward(loss_image, app->grid, H, W, app->grid_x, app->grid_y, app->grid_z, app->image,
                                                st)) != GSB_OK)
            return rc;
        sliced_image = app->image;
    }
    if (robust && (rc = launch_robust_pre(*robust, sliced_image, loss_gt, H, W, st)) != GSB_OK) return rc;
    rc = gsb200_image_loss(robust ? robust->composite : sliced_image, loss_gt, H, W, t->lambda_value, 1.0f, t->loss_out3,
                           const_cast<float *>(b.grad_rasterized_image), t->loss_temp, t->loss_temp_bytes, f.stream);
    if (rc != GSB_OK) return rc;
    // dL/dx' -> dL/dx of the image the loss read, before the slice backward and the supervision post-pass read it
    if (robust && (rc = launch_robust_post(*robust, sliced_image, H, W, const_cast<float *>(b.grad_rasterized_image), st)) !=
                      GSB_OK)
        return rc;
    // dL/dG from dL/dI'' before dL/dI' replaces it in the same buffer; then the TV term into dL/dG
    if (app && (rc = launch_bilateral_grid_backward(loss_image, app->grid, H, W, app->grid_x, app->grid_y, app->grid_z,
                                                    b.grad_rasterized_image, const_cast<float *>(b.grad_rasterized_image),
                                                    app->grad_grid, app->temp, app->tv_weight, app->loss_out1, st)) != GSB_OK)
        return rc;
    if (supervised && (rc = launch_supervision_post(*s, f.rasterized_image, t->ground_truth_image, f.pixel_accumulated_alpha,
                                                    f.rasterized_depth, H, W, b.grad_rasterized_image, t->loss_out3, st)) != GSB_OK)
        return rc;
    if (x && (rc = launch_feature_loss(*x, H, W, st)) != GSB_OK) return rc;
    if ((rc = backward_impl(&b, true, depth_on ? s->grad_depth : nullptr, depth_on ? f.rasterized_depth : nullptr,
                            alpha_on ? s->grad_pixel_accumulated_alpha : nullptr, ext, nullptr, nullptr, nullptr, nullptr,
                            nullptr, nullptr, filter3d)) != GSB_OK)
        return rc;
    Workspace ws;
    if ((rc = resolve_fwd(&f, &ws)) != GSB_OK) return rc;
    const long long *skip = ws.counters + CNT_OVERFLOW;
    if (mc && (rc = launch_mcmc_regulariser(f.pointcloud_features, f.point_invalid_mask, b.grad_pointcloud_features,
                                            f.num_points, mc->num_valid, mc->lambda_opacity, mc->lambda_scale, mc->terms_out2,
                                            mc->temp, skip, st)) != GSB_OK)
        return rc;
    rc = launch_adam_step(f.pointcloud_features, b.grad_pointcloud_features, t->feature_exp_avg, t->feature_exp_avg_sq,
                          (long long)f.num_points * GSB_FEATURE_DIM, t->feature_learning_rate, t->beta1, t->beta2, t->eps, t->step,
                          skip, st);
    if (rc != GSB_OK) return rc;
    rc = launch_adam_step(const_cast<float *>(f.pointcloud), b.grad_pointcloud, t->position_exp_avg, t->position_exp_avg_sq,
                          (long long)f.num_points * 3, t->position_learning_rate, t->beta1, t->beta2, t->eps, t->step, skip, st);
    if (rc != GSB_OK) return rc;
    if (x && (rc = launch_adam_step(const_cast<float *>(ext->features), ext->grad_features, x->exp_avg, x->exp_avg_sq,
                                    (long long)f.num_points * ext->channels, x->learning_rate, t->beta1, t->beta2, t->eps,
                                    t->step, skip, st)) != GSB_OK)
        return rc;
    if (app && (rc = launch_adam_step(app->grid, app->grad_grid, app->exp_avg, app->exp_avg_sq,
                                      12LL * app->grid_z * app->grid_y * app->grid_x, app->learning_rate, t->beta1, t->beta2,
                                      t->eps, app->step, skip, st)) != GSB_OK)
        return rc;
    if (!mc) return GSB_OK;
    return launch_mcmc_noise(const_cast<float *>(f.pointcloud), f.pointcloud_features, f.point_invalid_mask, f.num_points,
                             mc->noise_scale, mc->gate_k, mc->min_opacity, mc->seed, mc->step, skip, st);
}

int gsb200_expand_view_gradients(const GsbExpandArgs *a) {
    if (!a || a->num_points < 0 || a->num_views < 1 || a->num_objects < 1 || a->part < 0 || a->part > 2 ||
        (a->num_points > 0 && (!a->grad_sum || !a->grad_color_views || !a->pointcloud || !a->point_object_id ||
                               !a->grad_pointcloud || !a->grad_pointcloud_features)) ||
        a->view_stride < 3 * a->num_points + 3 * (int64_t)a->num_objects) {
        set_error("expand_view_gradients: bad arguments");
        return GSB_EINVAL;
    }
    if (reinterpret_cast<uintptr_t>(a->grad_sum) % 16 != 0 || reinterpret_cast<uintptr_t>(a->grad_pointcloud_features) % 16 != 0) {
        set_error("expand_view_gradients: grad_sum and grad_pointcloud_features must be 16-byte aligned");
        return GSB_EINVAL;
    }
    return launch_expand_view_gradients(*a, static_cast<cudaStream_t>(a->stream));
}

// ---- diagnostic variants: same launches as gsb200_forward / gsb200_backward with a CUDA event recorded
// on the launching stream between stages; returns device milliseconds per stage (host array of 8).
namespace {
struct StageTimer {
    cudaEvent_t ev[9];
    int n = 0;
    cudaStream_t st;
    bool ok = true;
    explicit StageTimer(cudaStream_t s) : st(s) {
        for (auto &e : ev) ok = ok && cudaEventCreate(&e) == cudaSuccess;
    }
    ~StageTimer() {
        for (auto &e : ev) cudaEventDestroy(e);
    }
    void mark() {
        if (n < 9) cudaEventRecord(ev[n++], st);
    }
    int finish(float *out) {
        if (cudaStreamSynchronize(st) != cudaSuccess) return GSB_ECUDA;
        for (int i = 0; i < 8; ++i) out[i] = 0.0f;
        for (int i = 0; i + 1 < n; ++i) cudaEventElapsedTime(&out[i], ev[i], ev[i + 1]);
        return GSB_OK;
    }
};
}  // namespace

int gsb200_forward_timed(const GsbForwardArgs *a, float *stage_ms_out) {
    Workspace ws;
    int rc = resolve_fwd(a, &ws);
    if (rc != GSB_OK) return rc;
    if (!stage_ms_out) return GSB_EINVAL;
    cudaStream_t st = static_cast<cudaStream_t>(a->stream);
    StageTimer t(st);
    if (!t.ok) {
        set_error("forward_timed: cudaEventCreate failed");
        return GSB_ECUDA;
    }
    const int T = (a->camera_height / GSB_TILE_HEIGHT) * (a->camera_width / GSB_TILE_WIDTH);
    t.mark();
    t.mark();  // the "memset" stage is empty: launch_preprocess's first kernel zeroes the per-frame state
    if ((rc = launch_preprocess(*a, ws, st)) != GSB_OK) return rc;
    t.mark();
    if ((rc = launch_sort(ws, a->key_capacity, st)) != GSB_OK) return rc;
    t.mark();
    if ((rc = launch_tile_ranges(ws, a->key_capacity, T, st)) != GSB_OK) return rc;
    t.mark();
    if ((rc = launch_blend_forward(*a, ws, st)) != GSB_OK) return rc;
    t.mark();
    return t.finish(stage_ms_out);
}

int gsb200_backward_timed(const GsbBackwardArgs *a, float *stage_ms_out) {
    if (!a || !stage_ms_out) return GSB_EINVAL;
    Workspace ws;
    int rc = resolve_workspace(a->workspace, a->workspace_bytes, a->num_points, a->num_objects,
                               a->key_capacity, a->camera_height, a->camera_width, a->far_plane,
                               a->depth_to_sort_key_scale, a->flags, &ws);
    if (rc != GSB_OK) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(a->stream);
    StageTimer t(st);
    if (!t.ok) {
        set_error("backward_timed: cudaEventCreate failed");
        return GSB_ECUDA;
    }
    t.mark();
    if (a->accum_rows > 0)
        GSB_CUDA_CHECK(cudaMemsetAsync(a->accum, 0, (size_t)a->accum_rows * GSB_ACCUM_FLOATS * 4, st));
    t.mark();
    if ((rc = launch_blend_backward(*a, ws, st)) != GSB_OK) return rc;
    t.mark();
    if ((rc = launch_backward_points(*a, ws, st)) != GSB_OK) return rc;
    t.mark();
    return t.finish(stage_ms_out);
}

int gsb200_forward_blend_work(const GsbForwardArgs *a, uint64_t *host_out8) {
    Workspace ws;
    int rc = resolve_fwd(a, &ws);
    if (rc != GSB_OK) return rc;
    if (!host_out8 || a->rgb_only) {
        set_error("forward_blend_work: host_out8 is null or rgb_only is set");
        return GSB_EINVAL;
    }
    cudaStream_t st = static_cast<cudaStream_t>(a->stream);
    unsigned long long *cnt = nullptr;  // a blocking diagnostic: its own small allocation
    GSB_CUDA_CHECK(cudaMalloc(&cnt, 64));
    cudaError_t e = cudaMemsetAsync(cnt, 0, 64, st);
    if (e == cudaSuccess) {
        rc = launch_blend_forward_count(*a, ws, cnt, st);
        if (rc == GSB_OK) e = cudaMemcpyAsync(host_out8, cnt, 64, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    }
    cudaFree(cnt);
    if (rc != GSB_OK) return rc;
    if (e != cudaSuccess) {
        set_error("forward_blend_work: %s", cudaGetErrorString(e));
        return GSB_ECUDA;
    }
    return GSB_OK;
}

int gsb200_backward_blend_work(const GsbBackwardArgs *a, uint64_t *host_out2) {
    if (!a || !host_out2 || !a->grad_rasterized_image || !a->pixel_accumulated_alpha ||
        !a->pixel_offset_of_last_effective_point || !a->accum) {
        set_error("backward_blend_work: null pointer argument");
        return GSB_EINVAL;
    }
    Workspace ws;
    int rc = resolve_workspace(a->workspace, a->workspace_bytes, a->num_points, a->num_objects,
                               a->key_capacity, a->camera_height, a->camera_width, a->far_plane,
                               a->depth_to_sort_key_scale, a->flags, &ws);
    if (rc != GSB_OK) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(a->stream);
    unsigned long long *cnt = reinterpret_cast<unsigned long long *>(ws.counters + 6);
    GSB_CUDA_CHECK(cudaMemsetAsync(cnt, 0, 16, st));
    if ((rc = launch_blend_backward_work(*a, ws, cnt, st)) != GSB_OK) return rc;
    GSB_CUDA_CHECK(cudaMemcpyAsync(host_out2, cnt, 16, cudaMemcpyDeviceToHost, st));
    GSB_CUDA_CHECK(cudaStreamSynchronize(st));
    return GSB_OK;
}

namespace {
__global__ void selftest_kernel(unsigned int *out) {
    float one = 1.0f, zero = 0.0f, r, e;
    asm volatile("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(one));
    asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(zero));
    out[0] = __float_as_uint(r);
    out[1] = __float_as_uint(e);
}
}  // namespace

int gsb200_device_selftest(void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    unsigned int *dev = nullptr, host[2] = {0u, 0u};
    GSB_CUDA_CHECK(cudaMalloc(&dev, 8));
    selftest_kernel<<<1, 1, 0, st>>>(dev);
    cudaError_t e = cudaMemcpyAsync(host, dev, 8, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    cudaFree(dev);
    if (e != cudaSuccess) {
        set_error("device_selftest: %s", cudaGetErrorString(e));
        return GSB_ECUDA;
    }
    if (host[0] != 0x3f800000u || host[1] != 0x3f800000u) {
        set_error("device_selftest: rcp.approx(1) = 0x%08x, ex2.approx(0) = 0x%08x (both must be 1.0f exactly)", host[0], host[1]);
        return GSB_EUNSUPPORTED;
    }
    return GSB_OK;
}

int gsb200_find_tile_start_and_end(const int64_t *sorted_keys, int64_t num_keys, int32_t *tile_points_start,
                                   int32_t *tile_points_end, int32_t num_tiles, void *stream) {
    if (num_keys < 0 || num_tiles < 0 || (num_keys > 0 && (!sorted_keys || !tile_points_start || !tile_points_end))) {
        set_error("find_tile_start_and_end: bad arguments");
        return GSB_EINVAL;
    }
    return launch_tile_ranges_raw(reinterpret_cast<const long long *>(sorted_keys), num_keys, tile_points_start,
                                  tile_points_end, num_tiles, static_cast<cudaStream_t>(stream));
}

int64_t gsb200_sort_temp_bytes(int64_t n, int32_t key_bytes) {
    const int64_t padded = align_up(n > 0 ? n : 1, SORT_TILE);
    const int64_t blocks = padded / SORT_TILE;
    int64_t off = 0;
    off += 256;                                      // n_dev
    off += 256;                                      // tickets
    off += 8 * 1024 * 4;                             // hist (up to 8 passes of up to 1024 bins)
    off += align_up(8 * blocks * 1024 * 4, 256);     // look-back state (up to 8 passes x 1024 digits)
    off += align_up(padded * key_bytes, 256);        // tmp keys
    off += align_up(padded * 4, 256);                // tmp vals
    return off;
}

int gsb200_sort_pairs(const void *keys_in, const int32_t *vals_in, void *keys_out, int32_t *vals_out,
                      int64_t n, int32_t key_bytes, int32_t end_bit, void *temp, int64_t temp_bytes,
                      void *stream) {
    if (n < 0 || (key_bytes != 4 && key_bytes != 8) || end_bit < 1 || end_bit > key_bytes * 8) {
        set_error("sort_pairs: bad arguments (n=%lld key_bytes=%d end_bit=%d)", (long long)n, key_bytes, end_bit);
        return GSB_EINVAL;
    }
    if (n == 0) return GSB_OK;
    if (n >= (1LL << 30)) {
        set_error("sort_pairs: n must be < 2^30");
        return GSB_EUNSUPPORTED;
    }
    if (!keys_in || !vals_in || !keys_out || !vals_out || !temp || temp_bytes < gsb200_sort_temp_bytes(n, key_bytes)) {
        set_error("sort_pairs: null pointer or temp too small");
        return GSB_EINVAL;
    }
    if (reinterpret_cast<uintptr_t>(keys_in) % 16 != 0 || reinterpret_cast<uintptr_t>(temp) % 256 != 0) {
        set_error("sort_pairs: keys_in must be 16-byte aligned and temp 256-byte aligned");
        return GSB_EINVAL;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int64_t padded = align_up(n, SORT_TILE);
    const int64_t blocks = padded / SORT_TILE;
    char *b = static_cast<char *>(temp);
    long long *n_dev = reinterpret_cast<long long *>(b);
    unsigned int *tickets = reinterpret_cast<unsigned int *>(b + 256);
    unsigned int *hist = reinterpret_cast<unsigned int *>(b + 512);
    unsigned int *state = reinterpret_cast<unsigned int *>(b + 512 + 8 * 1024 * 4);
    const int64_t state_bytes = align_up(8 * blocks * 1024 * 4, 256);
    void *tmp_keys = b + 512 + 8 * 1024 * 4 + state_bytes;
    int *tmp_vals = reinterpret_cast<int *>(static_cast<char *>(tmp_keys) + align_up(padded * key_bytes, 256));
    GSB_CUDA_CHECK(cudaMemsetAsync(b, 0, (size_t)(512 + 8 * 1024 * 4), st));  // n, tickets, hist; the sort clears its state
    const long long n_host = n;
    GSB_CUDA_CHECK(cudaMemcpyAsync(n_dev, &n_host, sizeof(n_host), cudaMemcpyHostToDevice, st));
    return sort_pairs_device(keys_in, vals_in, keys_out, vals_out, n_dev, padded, key_bytes, 0, end_bit, nullptr, hist,
                             state, tickets, tmp_keys, tmp_vals, st);
}

int gsb200_render_host(const GsbForwardArgs *device_args, const float *host_q, const float *host_t,
                       const float *host_K, float *staging, float *host_image_out,
                       int64_t *host_counters_out) {
    if (!device_args || !host_q || !host_t || !host_K || !staging || !host_image_out) {
        set_error("render_host: null pointer argument");
        return GSB_EINVAL;
    }
    GsbForwardArgs a = *device_args;
    cudaStream_t st = static_cast<cudaStream_t>(a.stream);
    const int n = a.num_objects;
    float *d_q = staging, *d_t = staging + 4 * n, *d_K = staging + 7 * n;
    GSB_CUDA_CHECK(cudaMemcpyAsync(d_q, host_q, sizeof(float) * 4 * n, cudaMemcpyHostToDevice, st));
    GSB_CUDA_CHECK(cudaMemcpyAsync(d_t, host_t, sizeof(float) * 3 * n, cudaMemcpyHostToDevice, st));
    GSB_CUDA_CHECK(cudaMemcpyAsync(d_K, host_K, sizeof(float) * 9, cudaMemcpyHostToDevice, st));
    a.q_pointcloud_camera = d_q;
    a.t_pointcloud_camera = d_t;
    a.camera_intrinsics = d_K;
    int rc = gsb200_forward(&a);
    if (rc != GSB_OK) return rc;
    GSB_CUDA_CHECK(cudaMemcpyAsync(host_image_out, a.rasterized_image,
                                   sizeof(float) * 3 * (size_t)a.camera_height * a.camera_width,
                                   cudaMemcpyDeviceToHost, st));
    if (host_counters_out)
        GSB_CUDA_CHECK(cudaMemcpyAsync(host_counters_out, a.workspace, sizeof(int64_t) * 4,
                                       cudaMemcpyDeviceToHost, st));
    GSB_CUDA_CHECK(cudaStreamSynchronize(st));
    return GSB_OK;
}

}  // extern "C"
