/*
 * gsb200.h -- C ABI of libgsb200.so: the H100-native (sm_90a) replacement for the rasteriser
 * hot path of wanmeihuali/taichi_3d_gaussian_splatting.
 *
 * This header is the drop-in boundary.  Every entry point names the reference interface it
 * replaces (file:line relative to the reference repo; GPCR =
 * taichi_3d_gaussian_splatting/GaussianPointCloudRasterisation.py).
 *
 * Conventions
 *  - extern "C", plain pointers and sizes only; no C++/torch types cross the boundary.
 *  - All pointers in the *Args structs are DEVICE pointers unless the field name says "host".
 *  - The caller owns every buffer, including the workspace; the library allocates nothing
 *    persistent and keeps no global mutable state except a thread-local error string.
 *  - Every call enqueues work on the given cudaStream_t (passed as void*) and returns without
 *    synchronising, except the *_host entry points which return after the result is in host memory.
 *  - Return value: 0 on success, negative GSB_E* code on failure; gsb200_last_error() gives text.
 *  - dtypes are the reference's: f32 data, i32 indices, i8 masks (GPCR:31-45, 239-259, 318-343).
 */
#ifndef GSB200_H_
#define GSB200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GSB200_VERSION 102 /* major*100 + minor */

#define GSB_TILE_WIDTH 16     /* GPCR:27 */
#define GSB_TILE_HEIGHT 16    /* GPCR:28 */
#define GSB_BOUNDARY_TILES 3  /* GPCR:26 */
#define GSB_FEATURE_DIM 56    /* GPCR:208-236: q(4) s(3) alpha(1) R/G/B SH(16 each) */
#define GSB_RECORD_FLOATS 12  /* packed per-splat record written by the preprocess kernel */
#define GSB_ACCUM_FLOATS 12   /* per-splat backward accumulator row */

enum {
    GSB_OK = 0,
    GSB_EINVAL = -1,     /* bad argument (null pointer, H/W not multiple of 16, ...) */
    GSB_ECUDA = -2,      /* a CUDA runtime call failed */
    GSB_EWORKSPACE = -3, /* workspace too small for (N, key_capacity, H, W) */
    GSB_EUNSUPPORTED = -4
};

/* flags */
#define GSB_FLAG_EXACT_EXP 1u    /* blend kernels use expf instead of ex2.approx */
#define GSB_FLAG_FORCE_KEY64 2u  /* always sort (tile<<32 | depth) 64-bit keys like GPCR:158-170 */
#define GSB_FLAG_KEEP_ALL_TILE_PAIRS 8u   /* emit a key for every tile of the reference's 3-sigma square (GPCR:81-172) instead of
                                            only those where the splat can reach alpha >= 1/255 on some pixel; outputs are
                                            identical either way, this only makes the sorted list equal to the reference's */
#define GSB_FLAG_Q_ALREADY_NORMALISED 4u /* forward only: take q as stored and do not rewrite it.  Used when a
                                            frame is re-run after a key-capacity overflow, so that the second
                                            pass is bit-identical to the first (normalising twice is not). */
#define GSB_FLAG_BACKWARD_TRANSPOSED 16u /* backward only: loop A accumulates per splat in registers after a shared-memory
                                            transposition (csrc/blend_bwd_transposed.cu; what the Python operator passes by
                                            default) instead of a warp butterfly per (warp, splat)
                                            (csrc/blend_bwd.cu; flag clear) */
#define GSB_FLAG_NO_HOOK_STATS 32u       /* backward only, opt-in: skip the statistics only a
                                            backward hook reads (|d/duv| magnitude, affected-pixel count, magnitude image) --
                                            the reference's need_extra_info = False, GPCR:521, 690-704.  accum[:, 9:11] and
                                            magnitude_grad_viewspace_on_image are then left untouched (the pointer must still be valid) */

#define GSB_FLAG_COMPACT_GRADS 64u        /* backward only (view-parallel training, parallel.py): the per-point kernel writes
                                            grad_sum_compact (N,12) and grad_color_compact (N,3) instead of the dense
                                            gradients; gsb200_expand_view_gradients rebuilds them after the exchange */

/* Byte offsets of the sub-buffers inside the caller-owned workspace blob.  Filled by
 * gsb200_workspace_layout(); the Python shim uses it to expose saved-for-backward tensors as views. */
typedef struct GsbWorkspaceLayout {
    int64_t total_bytes;
    int64_t zero_bytes;        /* [0, zero_bytes): per-frame state, cleared on the device by every forward's own kernels */
    int64_t counters;          /* int64[8]: [0]=M in-frustum points, [1]=K (tile,splat) pairs emitted/needed,
                                  [2]=overflow (K > key_capacity), [4]=largest depth key int32(depth * scale) of the frame
                                  (low 32 bits): the sort only runs the passes its live bits need */
    int64_t tickets;           /* uint32[16] dynamic block tickets */
    int64_t scan_state;        /* uint64[scan_blocks+1] decoupled look-back state of the compaction scan (one word per 128-point CTA) */
    int64_t sort_hist;         /* uint32[8][1024] global digit histograms */
    int64_t sort_state;        /* uint32[passes][sort_blocks][2^radix_bits] onesweep look-back state */
    int64_t tile_start;        /* int32[T]  GPCR:952-957 tile_points_start */
    int64_t tile_end;          /* int32[T]  tile_points_end */
    int64_t poses;             /* float[num_objects][20]: T_camera_pointcloud 3x4, camera centre, pad */
    int64_t point_id;          /* int32[N]  point_id_in_camera_list (first M valid), GPCR:864 */
    int64_t point_offset;      /* int32[N]  inverse map: in-camera offset of point id, -1 if outside the frustum */
    int64_t num_tiles;         /* int32[N]  num_overlap_tiles, GPCR:904-911 */
    int64_t records;           /* float[N][12]: u v a b | c rescale opacity depth | r g b radius */
    int64_t point_in_camera;   /* float[N][3] GPCR:877 */
    int64_t keys_a, keys_b;    /* sort keys, key_bytes each, key_capacity_padded entries: a = as emitted (never written by
                                  the sort), b = sorted (whatever the number of radix passes that ran) */
    int64_t vals_a, vals_b;    /* int32 payload = in-camera offset, GPCR:930 */
    int64_t keys_c, vals_c;    /* scratch of the radix passes (third buffer of the a -> [c -> b ->] ... -> b rotation) */
    int32_t key_bytes;         /* 4 or 8 */
    int32_t tile_bits, depth_bits, sort_passes;
    int64_t key_capacity_padded;
    int32_t sort_blocks, scan_blocks;
    int32_t radix_bits;        /* 8 or 10: digit width of the key sort */
    int32_t reserved;
} GsbWorkspaceLayout;

/* Inputs of GaussianPointCloudRasterisationInput (GPCR:788-804) + config (GPCR:776-786). */
typedef struct GsbForwardArgs {
    int64_t num_points;                 /* N */
    const float *pointcloud;            /* (N,3) */
    float *pointcloud_features;         /* (N,56); q of in-frustum rows normalised IN PLACE (GPCR:264-266) */
    const int8_t *point_invalid_mask;   /* (N) 1 = slot unused */
    const int32_t *point_object_id;     /* (N) */
    int32_t num_objects;
    const float *q_pointcloud_camera;   /* (num_objects,4) xyzw, camera->pointcloud */
    const float *t_pointcloud_camera;   /* (num_objects,3) */
    const float *camera_intrinsics;     /* (3,3) row-major, device */
    int32_t camera_height, camera_width;
    float near_plane, far_plane, depth_to_sort_key_scale;
    int32_t rgb_only;                   /* GPCR:781; aux outputs are left untouched when set */
    uint32_t flags;
    void *workspace;
    int64_t workspace_bytes;
    int64_t key_capacity;               /* capacity (entries) of the key/value buffers */
    float *rasterized_image;            /* (H,W,3) */
    float *rasterized_depth;            /* (H,W) */
    float *pixel_accumulated_alpha;     /* (H,W) */
    int32_t *pixel_offset_of_last_effective_point; /* (H,W) */
    int32_t *pixel_valid_point_count;   /* (H,W) */
    void *stream;
    /* Optional early read-back: if both are non-NULL, gsb200_forward copies counters[0..3] = {M, K, overflow, -}
     * to the PINNED HOST buffer right after the per-point stage and records the event (a cudaEvent_t) behind
     * the copy; the remaining stages are enqueued regardless.  The host can wait on the event (it fires after
     * ~the preprocess kernel, long before the frame ends), learn M and K and whether the key buffers overflowed,
     * and return to its caller with the rest of the frame still in flight. */
    int64_t *host_counters;
    void *host_counters_event;
} GsbForwardArgs;

typedef struct GsbBackwardArgs {
    int64_t num_points;
    const float *pointcloud;
    const float *pointcloud_features;   /* as left by forward (q normalised) */
    const int32_t *point_object_id;
    int32_t num_objects;
    const float *t_pointcloud_camera;   /* camera centre for the SH direction, GPCR:731-732 */
    const float *camera_intrinsics;
    int32_t camera_height, camera_width;
    float far_plane, depth_to_sort_key_scale; /* same values as the forward (fix the workspace layout) */
    int32_t color_max_sh_band;          /* GPCR:1167-1182; any value outside {0,1,2} clears nothing */
    float grad_q_factor, grad_s_factor, grad_alpha_factor, grad_color_factor,
        grad_high_order_color_factor;   /* GPCR:782-786, 1105-1125 */
    uint32_t flags;
    void *workspace;                    /* the SAME workspace the forward of this frame used */
    int64_t workspace_bytes;
    int64_t key_capacity;
    const float *grad_rasterized_image; /* (H,W,3) */
    const float *pixel_accumulated_alpha;
    const int32_t *pixel_offset_of_last_effective_point;
    float *accum;                       /* (>=M,12) zero-initialised by this call:
                                           guv.x guv.y gcov00 gcov01 gcov11 gr gg gb glogit magnitude n_pixels(as f32) pad */
    int64_t accum_rows;
    float *grad_pointcloud;             /* (N,3) fully written by the per-point kernel (zeros outside the frustum) */
    float *grad_pointcloud_features;    /* (N,56) fully written, band-masked and factor-scaled */
    float *magnitude_grad_viewspace_on_image; /* (H,W,2) */
    void *stream;
    /* GSB_FLAG_COMPACT_GRADS only (then grad_pointcloud / grad_pointcloud_features may be NULL): per scene row, zeros outside
     * the frustum -- grad_sum_compact (N,12) = xyz(3) q(4) s(3) logit(1) pad, factors applied: the columns that add up over
     * views; grad_color_compact (N,3) = dL/d(SH colour argument) of THIS view (its 48 SH gradients are the outer product
     * with this view's SH basis, GPCR:749-756). */
    float *grad_sum_compact;
    float *grad_color_compact;
    /* Optional, all NULL or all set: the densification controller's accumulators (GaussianPointAdaptiveController.py:108-116),
     * updated for every in-camera point in the epilogue of the per-point kernel exactly as GaussianPointAdaptiveController.update
     * does from the hook tensors (:130-143) -- no gathers, no extra launch.  (N) each, accumulated_position_gradients (N,3). */
    int32_t *ctl_accumulated_num_in_camera;
    int32_t *ctl_accumulated_num_pixels;
    float *ctl_accumulated_view_space_position_gradients;
    float *ctl_accumulated_view_space_position_gradients_avg;
    float *ctl_accumulated_position_gradients;
    float *ctl_accumulated_position_gradients_norm;
} GsbBackwardArgs;

/* View-parallel training (SURVEY 8(e); the reference is single-GPU): after the ranks have exchanged their COMPACT rows --
 * all-reduce(sum) of grad_sum_compact, all-gather of [grad_color_compact | t_pointcloud_camera] -- rebuild the dense
 * gradients of the whole batch of views: (N,3) and (N,56) exactly as the sum over views of what gsb200_backward writes
 * per view (SH gradient of view v = colour-argument gradient (x) SH basis along xyz - camera centre of v, times the
 * colour factors, masked by color_max_sh_band; GPCR:749-756, 1105-1125, 1167-1182), summed in view order.
 * 14 instead of 59 floats per Gaussian cross NVLink. */
typedef struct GsbExpandArgs {
    int64_t num_points;
    int32_t num_views, num_objects;
    const float *grad_sum;          /* (N,12), already summed over the views */
    const float *grad_color_views;  /* num_views blocks, view_stride floats apart: [N*3 colour-argument gradients |
                                       num_objects*3 camera centres (that view's t_pointcloud_camera)] */
    int64_t view_stride;            /* >= 3*N + 3*num_objects */
    const float *pointcloud;        /* (N,3) */
    const int32_t *point_object_id; /* (N) */
    int32_t color_max_sh_band;
    float grad_color_factor, grad_high_order_color_factor;
    int32_t part;                    /* 0: everything.  1: only the 48 SH columns (reads the blocks, not grad_sum); 2: only xyz and the
                                        q / s / logit columns (reads grad_sum, not the blocks).  1 and 2 write disjoint pieces of
                                        the outputs, so 1 can run on another stream while the all-reduce of grad_sum is in flight */
    float *grad_pointcloud;          /* (N,3) out */
    float *grad_pointcloud_features; /* (N,56) out */
    void *stream;
} GsbExpandArgs;

/* version / errors */
int gsb200_version(void);
const char *gsb200_last_error(void);
/* sizeof(GsbWorkspaceLayout), sizeof(GsbForwardArgs), sizeof(GsbBackwardArgs) as compiled: lets a
 * foreign-language binding verify its struct mirrors. */
void gsb200_abi_sizes(int64_t *out3);
/* ... and of the first n of {GsbWorkspaceLayout, GsbForwardArgs, GsbBackwardArgs, GsbExpandArgs, GsbTrainStepArgs,
 * GsbSupervisionArgs, GsbExtraFeatureArgs, GsbFeatureTrainArgs, GsbPoseGradArgs, GsbIntrinsicsGradArgs, GsbLensArgs,
 * GsbLensGradArgs, GsbRollingShutterArgs, GsbRollingShutterGradArgs, GsbAppearanceArgs} */
void gsb200_abi_sizes_ext(int64_t *out, int32_t n);
/* sizeof(GsbMcmcRelocateArgs), sizeof(GsbMcmcStepArgs).  A call of their own: the table of gsb200_abi_sizes_ext ends at
 * GsbAppearanceArgs, and a binding may rely on slots past its end staying untouched. */
void gsb200_abi_sizes_mcmc(int64_t *out2);

/* Workspace sizing.  far_plane*depth_to_sort_key_scale fixes the depth-key width; (H/16)*(W/16)
 * the tile-id width; both <= 32 bits total selects 32-bit sort keys.
 * Limits (GSB_EUNSUPPORTED beyond them): num_points < 2^26, key_capacity < 2^30.  The single-pass scan of the per-point stage
 * carries (in-camera count, pair count) in one 64-bit word with 26 + 36 bits: a frame whose REFERENCE pair count (sum of
 * num_overlap_tiles, before the reach filter and regardless of key_capacity) reached 2^36 = 6.9e10 would carry into the
 * point count -- such a frame needs > 0.8 TB of keys in the reference and is far beyond key_capacity < 2^30, but it is the
 * caller's responsibility not to submit one (e.g. millions of screen-filling splats at 4K). */
int gsb200_workspace_layout(int64_t num_points, int32_t num_objects, int64_t key_capacity,
                            int32_t camera_height, int32_t camera_width, float far_plane,
                            float depth_to_sort_key_scale, uint32_t flags,
                            GsbWorkspaceLayout *out);

/* Forward: replaces _module_function.forward, GPCR:830-1023 (K1 filter_point_in_camera GPCR:31-78,
 * mask compaction GPCR:861-864, K2 generate_point_attributes_in_camera_plane GPCR:239-315,
 * K3 generate_num_overlap_tiles GPCR:106-128, cumsum GPCR:913-922,
 * K4 generate_point_sort_key_by_num_overlap_tiles GPCR:131-172, sort GPCR:947-950,
 * K5 find_tile_start_and_end GPCR:175-193, K6 gaussian_point_rasterisation GPCR:318-485). */
int gsb200_forward(const GsbForwardArgs *args);

/* Backward: replaces _module_function.backward, GPCR:1025-1125 (K7
 * gaussian_point_rasterisation_backward GPCR:488-772, _clear_grad_by_color_max_sh_band
 * GPCR:1167-1182, factor scaling GPCR:1105-1125). */
int gsb200_backward(const GsbBackwardArgs *args);

/* gsb200_backward for a loss on the image AND the depth map (an extension: the reference's depth output is not
 * differentiable).  With D = sum w z / S (S = sum w = pixel_accumulated_alpha) the depth gradient flows through alpha into
 * uv, conic and opacity like a fourth colour channel with "colour" z - D, and directly into xyz along the camera's viewing
 * axis.  Both pointers NULL: exactly gsb200_backward.  Exactly one NULL: GSB_EINVAL.  Depth without
 * GSB_FLAG_BACKWARD_TRANSPOSED (the butterfly kernel does not implement it): GSB_EUNSUPPORTED.  These checks come before any
 * CUDA call.  The accumulator rows carry dL/dz in their last word.  Same as gsb200_backward_aux(args, grad, depth, NULL). */
int gsb200_backward_with_depth(const GsbBackwardArgs *args,
                               const float *grad_rasterized_depth, /* (H,W) f32, device */
                               const float *rasterized_depth);     /* (H,W) f32: this frame's forward output */

/* gsb200_backward for a loss on the image and any of the other per-pixel float outputs (an extension: the reference
 * differentiates the image alone).  The depth pair follows gsb200_backward_with_depth.  grad_pixel_accumulated_alpha is
 * dL/dS for S = pixel_accumulated_alpha = 1 - prod (1 - alpha): S is the blend of a colour channel whose colour is 1
 * (dS/dalpha_i = T_final / (1 - alpha_i)), so its gradient flows through alpha into uv, conic and opacity; NULL means no
 * alpha term.  All three NULL: exactly gsb200_backward.  Depth pair with exactly one NULL: GSB_EINVAL.  Any term without
 * GSB_FLAG_BACKWARD_TRANSPOSED (the butterfly kernel implements neither): GSB_EUNSUPPORTED.  These checks come before any
 * CUDA call. */
int gsb200_backward_aux(const GsbBackwardArgs *args,
                        const float *grad_rasterized_depth,         /* (H,W) f32, device, or NULL */
                        const float *rasterized_depth,              /* (H,W) f32: this frame's forward output, or NULL */
                        const float *grad_pixel_accumulated_alpha); /* (H,W) f32, device, or NULL */

/* Per-Gaussian feature vectors rendered and differentiated alongside the image (an extension: the reference blends the SH
 * colour alone).  C values per Gaussian, chosen by the caller (semantic logits, instance encodings, distilled features),
 * are blended with exactly the image's weights w_i = alpha_i T_i -- the 1/255 cut, the 0.99 clamp and the 1e-4 stop
 * included -- into F_p = sum_i w_i f_i: no normalisation, no background, no activation.  Rows of invalid or out-of-frustum
 * points never contribute.  All pointers are device memory, rows contiguous. */
typedef struct GsbExtraFeatureArgs {
    int32_t channels;              /* C, 1..16 */
    const float *features;         /* (N,C) f32, indexed by scene row like pointcloud */
    float *rasterized;             /* (H,W,C) f32: forward output */
    const float *grad_rasterized;  /* (H,W,C) f32: backward input dL/dF */
    float *grad_features;          /* (N,C) f32: backward output dL/df, fully written (zero for rows outside the frustum);
                                      16-byte aligned */
} GsbExtraFeatureArgs;

/* gsb200_forward that also blends the feature vectors of `ext` into ext->rasterized (features / rasterized must be set;
 * grad_* are not read).  NULL ext: exactly gsb200_forward (which is this call with NULL).  GSB_EINVAL, before any CUDA call,
 * for channels outside 1..16, a NULL features / rasterized pointer or rgb_only.  Every other output of the frame is
 * bit-identical to gsb200_forward's on the default arithmetic. */
int gsb200_forward_ext(const GsbForwardArgs *args, const GsbExtraFeatureArgs *ext);

/* gsb200_backward_aux that also back-propagates the feature map's gradient ext->grad_rasterized: dL/df_i = sum_p w_{p,i}
 * dL/dF_p into ext->grad_features (zeroed by the call, no gradient factor), and the feature loss's share of dL/dalpha into
 * uv, conic and opacity -- and from there into the hook statistics and the controller accumulators -- exactly as the image
 * loss's share.  In the backward each feature channel is one more colour channel of the blend.  NULL ext: exactly
 * gsb200_backward_aux (which is this call with NULL).  With ext, before any CUDA call: GSB_EINVAL for channels outside 1..16
 * or a NULL features / grad_rasterized / grad_features pointer; GSB_EUNSUPPORTED without GSB_FLAG_BACKWARD_TRANSPOSED
 * (the butterfly kernel does not implement it) or with GSB_FLAG_COMPACT_GRADS (the view-parallel exchange does not carry
 * the feature rows).  ext->features must be the rows the forward of this frame blended. */
int gsb200_backward_ext(const GsbBackwardArgs *args,
                        const float *grad_rasterized_depth,          /* as gsb200_backward_aux */
                        const float *rasterized_depth,
                        const float *grad_pixel_accumulated_alpha,
                        const GsbExtraFeatureArgs *ext);             /* or NULL */

/* Camera-pose gradients (an extension: the reference differentiates the scene only).  pose_kernel (csrc/preprocess.cu)
 * maps (q_pc, t_pc) of object o to T = [W | tw] with qi = conj(q_pc), W = R(qi) (the GP3D:30-48 polynomial on the
 * components as given) and tw = -R(qn) t_pc, qn = qi / |qi|; a point of the object is at pc = W xyz + tw in the camera.
 * The pose gradient is the exact derivative of the rendered outputs with respect to q_pc and t_pc through this map, under
 * the conventions of the point gradients: J inside Sigma' = J W Sigma W^T J^T, the SH view direction and the rescale factor
 * are detached, the 0.99 clamp is straight-through.  Per in-camera point, with gp = dL/dpc (through uv by the full-K
 * projection Jacobian, plus dL/dz of the depth term) and G the (g00, g01, g11) weighting of dL/dSigma':
 *   dL/dW += gp xyz^T + 2 J^T G (J W) Sigma,   dL/dtw += gp,
 * summed per object and taken through the map above.  No gradient factor is applied; every loss term the backward takes
 * (image, depth, alpha, features) contributes.  For one object with a unit q_pc, dL/dt_pc = -sum_i dL/dxyz_i.
 * The sum is deterministic: the per-point kernel runs on min(ceil(N/128), GSB_POSE_PARTIAL_BLOCKS) CTAs, each writes its
 * per-object sums to `temp` in a fixed order, and a second kernel adds them in block order -- no float atomics. */
#define GSB_POSE_MAX_OBJECTS 64        /* per-warp pose rows live in shared memory */
#define GSB_POSE_PARTIAL_BLOCKS 2048
typedef struct GsbPoseGradArgs {
    const float *q_pointcloud_camera;  /* (num_objects,4): the forward's input */
    float *grad_q_pointcloud_camera;   /* (num_objects,4) out, fully written */
    float *grad_t_pointcloud_camera;   /* (num_objects,3) out, fully written */
    void *temp;                        /* gsb200_pose_grad_temp_bytes(num_objects) bytes, 16-byte aligned */
} GsbPoseGradArgs;
/* GSB_POSE_PARTIAL_BLOCKS * num_objects * 12 floats (0 for num_objects < 1) */
int64_t gsb200_pose_grad_temp_bytes(int32_t num_objects);
/* gsb200_backward_ext that also writes the pose gradients of `pose`.  Everything else the call writes (dense gradients,
 * hook tensors, controller accumulators) is bit-identical to gsb200_backward_ext's.  NULL pose: exactly
 * gsb200_backward_ext.  With pose, before any CUDA call: GSB_EINVAL for a NULL q / output / temp pointer, a temp that is
 * not 16-byte aligned or num_objects < 1; GSB_EUNSUPPORTED for num_objects > GSB_POSE_MAX_OBJECTS or
 * GSB_FLAG_COMPACT_GRADS.  An image-only loss works with either loop-A kernel; the other terms keep their requirement of
 * GSB_FLAG_BACKWARD_TRANSPOSED. */
int gsb200_backward_pose(const GsbBackwardArgs *args, const float *grad_rasterized_depth, const float *rasterized_depth,
                         const float *grad_pixel_accumulated_alpha, const GsbExtraFeatureArgs *ext,
                         const GsbPoseGradArgs *pose); /* or NULL */

/* Camera-intrinsics gradients (an extension: the reference differentiates the scene only).  The forward (preprocess.cu)
 * reads K in two places: uv = (K pc)[:2] / z, which uses all six entries of rows 0 and 1, and J = [fx/z 0 -fx x/z^2;
 * 0 fy/z -fy y/z^2] (fx = K[0][0], fy = K[1][1]; skew does not enter J) inside Sigma' = (J W) Sigma (J W)^T.  Row 2 is never
 * read.  The intrinsics gradient is the exact derivative through both, under the conventions of the point and pose
 * gradients: the dependence of J on pc is detached, so are the rescale factor, the radius and tile membership and the SH
 * view direction; the 0.99 clamp is straight-through.  Per in-camera point, with guv = dL/duv of its accumulator row and
 * B0, B1 the rows of G (J W) Sigma (the pose gradient's):
 *   dL/dK[r][c] += guv_r pc_c / z                                 r in {0,1}, c in {0,1,2}
 *   dL/dK[0][0] += 2 sum_c B0[c] (W[0][c]/z - x W[2][c]/z^2),   dL/dK[1][1] += 2 sum_c B1[c] (W[1][c]/z - y W[2][c]/z^2)
 * summed over every in-camera point of every object (a frame has one K); dL/dK[2][.] = 0.  No gradient factor is applied;
 * every loss term that reaches the accumulator rows (image, depth, alpha, features) contributes, and the depth term's direct
 * dL/dz adds nothing (z does not depend on K).  The sum is deterministic: the per-point kernel runs on
 * min(ceil(N/128), GSB_INTRINSICS_PARTIAL_BLOCKS) CTAs, each writes its sums to `temp`, and a second kernel adds them in
 * block order -- no float atomics. */
#define GSB_INTRINSICS_PARTIAL_BLOCKS 2048 /* = GSB_POSE_PARTIAL_BLOCKS: with both, one per-point pass */
typedef struct GsbIntrinsicsGradArgs {
    float *grad_camera_intrinsics; /* (3,3) out, fully written (row 2 zero) */
    void *temp;                    /* gsb200_intrinsics_grad_temp_bytes() bytes, 16-byte aligned */
} GsbIntrinsicsGradArgs;
/* GSB_INTRINSICS_PARTIAL_BLOCKS * 6 floats */
int64_t gsb200_intrinsics_grad_temp_bytes(void);
/* gsb200_backward_pose that also writes the intrinsics gradient of `intrinsics`; with a pose as well, both come from one
 * pass of the per-point kernel.  Everything else the call writes (dense gradients, hook tensors, controller accumulators,
 * the pose gradients) is bit-identical to gsb200_backward_pose's.  NULL intrinsics: exactly gsb200_backward_pose, with the
 * same kernels.  With intrinsics, before any CUDA call: GSB_EINVAL for a NULL output or temp pointer or a temp that is not
 * 16-byte aligned; GSB_EUNSUPPORTED for GSB_FLAG_COMPACT_GRADS.  An image-only loss works with either loop-A kernel; the
 * other terms keep their requirement of GSB_FLAG_BACKWARD_TRANSPOSED. */
int gsb200_backward_calib(const GsbBackwardArgs *args, const float *grad_rasterized_depth, const float *rasterized_depth,
                          const float *grad_pixel_accumulated_alpha, const GsbExtraFeatureArgs *ext,
                          const GsbPoseGradArgs *pose,               /* or NULL */
                          const GsbIntrinsicsGradArgs *intrinsics);  /* or NULL */

/* Lens distortion (an extension: the reference projects through a pinhole).  The lens acts between the camera-frame point
 * pc = (x, y, z) and K.  With xn = x/z, yn = y/z, r^2 = xn^2 + yn^2:
 *   GSB_LENS_OPENCV (k1 k2 p1 p2 k3, OpenCV's distCoeffs order; COLMAP SIMPLE_RADIAL, RADIAL, OPENCV):
 *     rad = 1 + k1 r^2 + k2 r^4 + k3 r^6,  xd = xn rad + 2 p1 xn yn + p2 (r^2 + 2 xn^2),  yd = yn rad + p1 (r^2 + 2 yn^2) + 2 p2 xn yn
 *   GSB_LENS_FISHEYE (equidistant, k1 k2 k3 k4; COLMAP OPENCV_FISHEYE, cv2.fisheye; coefficients[4] must be 0):
 *     theta = atan(r),  theta_d = theta (1 + k1 theta^2 + k2 theta^4 + k3 theta^6 + k4 theta^8),  (xd, yd) = (theta_d / r) (xn, yn)
 *     (theta_d / r -> 1 on the optical axis; a series is used for small r)
 *   u = K00 xd + K01 yd + K02,  v = K10 xd + K11 yd + K12   (today's (K pc)[:2] / z with (xn, yn) replaced by (xd, yd)).
 * The covariance uses J = diag(fx, fy) D P with D = d(xd, yd)/d(xn, yn) and P = [1/z 0 -x/z^2; 0 1/z -y/z^2] (D = I is the
 * pinhole J); the 0.3 low-pass, rescale, radius, bounding box and reach filter follow from Sigma' as for a pinhole.
 * Validity: the radial map folds back beyond r_max -- for opencv the smallest positive root of 1 + 3 k1 r^2 + 5 k2 r^4 +
 * 7 k3 r^6 (tangential terms ignored; none: unbounded), for fisheye tan(min(pi/2, smallest positive root of dtheta_d/dtheta)).
 * The bound is computed once per call on the host in double and applied as an r^2 bound: a point with r^2 > r_max^2 is
 * outside the frustum (no key, point_offset -1, zero gradient).  The near / far / image-border tests apply to the distorted
 * (u, v).  Gradients: d uv / d pc = K[:2,:2] D P exactly; Sigma' uses the lens J; the conventions of the point gradients
 * hold (J's dependence on pc, the SH view direction and rescale detached, the 0.99 clamp straight-through, the validity cut
 * not differentiated).  The gradient with respect to the coefficients is opt-in: gsb200_backward_lens_grad below. */
#define GSB_LENS_PINHOLE 0
#define GSB_LENS_OPENCV 1
#define GSB_LENS_FISHEYE 2
typedef struct GsbLensArgs {
    int32_t model;          /* GSB_LENS_* */
    float coefficients[5];  /* opencv: k1 k2 p1 p2 k3; fisheye: k1 k2 k3 k4 0 */
} GsbLensArgs;
/* gsb200_forward_ext through the lens of `lens`.  NULL lens or GSB_LENS_PINHOLE: exactly gsb200_forward_ext.  Before any
 * CUDA call: GSB_EINVAL for an unknown model, a non-finite coefficient or a non-zero unused coefficient. */
int gsb200_forward_lens(const GsbForwardArgs *args, const GsbExtraFeatureArgs *ext, const GsbLensArgs *lens);
/* gsb200_backward_ext of a frame rendered by gsb200_forward_lens with the same lens.  NULL lens or GSB_LENS_PINHOLE: exactly
 * gsb200_backward_ext.  Before any CUDA call: the lens checks of gsb200_forward_lens, and GSB_EUNSUPPORTED with
 * GSB_FLAG_COMPACT_GRADS (the view-parallel exchange does not rebuild lens gradients).  An image-only loss works with either
 * loop-A kernel; the other terms keep their requirement of GSB_FLAG_BACKWARD_TRANSPOSED. */
int gsb200_backward_lens(const GsbBackwardArgs *args, const float *grad_rasterized_depth, const float *rasterized_depth,
                         const float *grad_pixel_accumulated_alpha, const GsbExtraFeatureArgs *ext,
                         const GsbLensArgs *lens);  /* or NULL */

/* Equirectangular 360-degree panoramas (an extension: the reference projects through a pinhole).  Camera frame as everywhere
 * (x right, y down, z forward).  With rho = sqrt(x^2 + z^2) and r = sqrt(rho^2 + y^2):
 *   lon = atan2(x, z),  lat = atan2(y, rho),  u = K00 lon + K02 reduced into [0, W),  v = K11 lat + K12.
 * A full panorama has K00 = W / 2pi, K11 = H / pi, K02 = W / 2, K12 = H / 2; the image centre looks along +z.
 * Covariance: Sigma' = J W Sigma W^T J^T with J = diag(K00, K11) [z/rho^2 0 -x/rho^2; -x y/(r^2 rho) rho/r^2 -z y/(r^2 rho)]
 * (the local affine projection); the 0.3 low-pass, rescale, 3-sigma radius and reach filter are the pinhole's.
 * In view: near < r < far and rho > GSB_EQUIRECT_POLE_EPSILON r (a cone of half-angle ~0.057 degrees around each pole, where
 * lon is undefined, is culled).  Points behind the camera are in view.  The depth is the ray distance r: in the sort key,
 * the record's depth slot, the depth output and the hook's point_depth.
 * Seam: the footprint's tile columns are not clamped to the image; a footprint wider than the panorama is cut to the W/16
 * columns whose centres lie within W/2 of u.  The reach filter runs in these unwrapped columns, and the key's tile column is
 * taken modulo W/16.  The blend kernels stage each splat at the copy of u nearest the tile's centre column,
 * u + W rint((tile centre - u) / W); the per-pixel arithmetic is unchanged, and dL/du does not change under the shift.
 * Gradients: d(u, v)/d pc = J exactly (J's dependence on pc detached inside Sigma', as for every model); the depth gradient
 * enters pc along pc / r.  Known limit: the affine approximation degrades towards the poles, where a Gaussian is drawn across
 * up to the full width of its rows; outputs and gradients stay finite there. */
#define GSB_EQUIRECT_POLE_EPSILON 1e-3f
/* |2 pi K00 - W| <= GSB_EQUIRECT_FX_TOLERANCE W: the panorama covers 360 degrees */
#define GSB_EQUIRECT_FX_TOLERANCE 1e-4f
/* gsb200_forward_ext of an equirectangular view.  Before any kernel runs: GSB_EINVAL when W is not a multiple of 16 or for
 * the checks of gsb200_forward_ext; then K (device memory, like every call's) is read back -- 36 bytes and one
 * synchronisation of args->stream -- and GSB_EINVAL when |2 pi K00 - W| > GSB_EQUIRECT_FX_TOLERANCE W, K01 or K10 is not 0,
 * K's last row is not (0, 0, 1), or an entry is not finite. */
int gsb200_forward_equirect(const GsbForwardArgs *args, const GsbExtraFeatureArgs *ext);
/* gsb200_backward_ext of a frame rendered by gsb200_forward_equirect.  The checks of gsb200_forward_equirect, and before any
 * CUDA call GSB_EUNSUPPORTED with GSB_FLAG_COMPACT_GRADS (the view-parallel exchange) or without
 * GSB_FLAG_BACKWARD_TRANSPOSED (the butterfly loop A does not wrap the seam). */
int gsb200_backward_equirect(const GsbBackwardArgs *args, const float *grad_rasterized_depth, const float *rasterized_depth,
                             const float *grad_pixel_accumulated_alpha, const GsbExtraFeatureArgs *ext);

/* Lens-coefficient gradients (an extension).  The forward is gsb200_forward_lens, unchanged; it reads the coefficients in
 * two places: the position u = K00 xd + K01 yd + K02, v = K10 xd + K11 yd + K12, and D = d(xd, yd)/d(xn, yn) inside
 * J = diag(fx, fy) D P, Sigma' = (J W) Sigma (J W)^T.  The coefficient gradient is the exact derivative through both, under
 * the conventions of the point, pose and intrinsics gradients: D is evaluated at the detached point but differentiated with
 * respect to k; rescale, the radius, tile membership and the SH view direction are detached; the r_max validity cut is not
 * differentiated (r_max is recomputed from the coefficients of each call); the 0.99 clamp is straight-through.  Per
 * in-camera point, with guv = dL/duv of its accumulator row and B0, B1 the rows of G (J W) Sigma (so dL/d(J W) = 2 [B0; B1]):
 *   dL/dk_i += guv^T K[:2,:2] d(xd, yd)/dk_i
 *   dL/dJ = 2 [B0; B1] W^T,  dL/dD = diag(fx, fy) dL/dJ P^T,  dL/dk_i += <dL/dD, dD/dk_i>
 * summed over every in-camera point of every object.  d(xd, yd)/dk and dD/dk are closed forms (lens_coefficient_grad in
 * csrc/common.cuh): opencv d(xd, yd)/dk1 = r^2 (xn, yn), /dk2 = r^4 (xn, yn), /dk3 = r^6 (xn, yn), /dp1 = (2 xn yn,
 * r^2 + 2 yn^2), /dp2 = (r^2 + 2 xn^2, 2 xn yn); fisheye with t = theta^2 and s = theta_d / r = A P(t): ds/dk_j = A t^j,
 * dg/dk_j = (A'/r) t^j + 2 A^2 j t^(j-1) / (1 + r^2) for D = s I + g (xn, yn)^T (xn, yn).  No gradient factor is applied;
 * every loss term that reaches the accumulator rows (image, depth, alpha, features) contributes, and the depth term's direct
 * dL/dz adds nothing (z does not depend on k).  The sum is deterministic: the per-point kernel runs on
 * min(ceil(N/128), GSB_LENS_GRAD_PARTIAL_BLOCKS) CTAs, each writes its sums to `temp`, and a second kernel adds them in block
 * order -- no float atomics. */
#define GSB_LENS_GRAD_PARTIAL_BLOCKS 2048
typedef struct GsbLensGradArgs {
    float *grad_coefficients; /* (5,) out, fully written in GsbLensArgs::coefficients' order; unused slots 0 */
    void *temp;               /* gsb200_lens_grad_temp_bytes() bytes, 16-byte aligned */
} GsbLensGradArgs;
/* GSB_LENS_GRAD_PARTIAL_BLOCKS * 5 floats */
int64_t gsb200_lens_grad_temp_bytes(void);
/* gsb200_backward_lens that also writes the coefficient gradient of `lens` to `lens_grad`.  Everything else the call writes
 * (dense gradients, hook tensors, controller accumulators) is bit-identical to gsb200_backward_lens's.  NULL lens_grad:
 * exactly gsb200_backward_lens.  With lens_grad, before any CUDA call: the lens checks of gsb200_forward_lens; GSB_EINVAL for a
 * NULL or pinhole lens, a NULL output or temp pointer, an output that is not 4-byte aligned or a temp that is not 16-byte
 * aligned; GSB_EUNSUPPORTED for GSB_FLAG_COMPACT_GRADS.  An image-only loss works with either loop-A kernel; the other terms
 * keep their requirement of GSB_FLAG_BACKWARD_TRANSPOSED. */
int gsb200_backward_lens_grad(const GsbBackwardArgs *args, const float *grad_rasterized_depth, const float *rasterized_depth,
                              const float *grad_pixel_accumulated_alpha, const GsbExtraFeatureArgs *ext,
                              const GsbLensArgs *lens, const GsbLensGradArgs *lens_grad); /* lens_grad or NULL */

/* Pose and intrinsics gradients through a lens (an extension): photometric self-calibration of OpenCV and fisheye cameras.
 * The forward is gsb200_forward_lens, unchanged.  The conventions are those of the point, pose, intrinsics and coefficient
 * gradients: J's dependence on pc is detached, D is evaluated at the detached point, rescale, the radius, tile membership
 * and the SH view direction are detached, the r_max validity cut is not differentiated and the 0.99 clamp is
 * straight-through.  Per in-camera point, with gp = dL/dpc (through uv by K[:2,:2] D P, plus dL/dz of the depth term),
 * guv = dL/duv of its accumulator row and B0, B1 the rows of G (J W) Sigma with the lens J = diag(fx, fy) D P:
 *   pose:        dL/dW += gp xyz^T + 2 J^T G (J W) Sigma,   dL/dtw += gp
 *                (gsb200_backward_pose's formula with the lens J and gp; summed per object, then taken to (q_pc, t_pc))
 *   intrinsics:  dL/dK[r][c] += guv_r (xd, yd, 1)_c                    r in {0,1}, c in {0,1,2}
 *                dL/dK[0][0] += 2 sum_c B0[c] (D P W)[0][c],   dL/dK[1][1] += 2 sum_c B1[c] (D P W)[1][c],   row 2 is 0
 *                (with D = I: gsb200_backward_calib's formula)
 *   coefficients: gsb200_backward_lens_grad's.
 * With any of the three, all of them come from one pass of one per-point kernel, whose per-CTA sums go to the three temps,
 * and the three finishing kernels of gsb200_backward_pose, gsb200_backward_calib and gsb200_backward_lens_grad add them in
 * block order -- no float atomics. */
/* gsb200_backward_lens_grad that also writes the pose gradients of `pose` and the intrinsics gradient of `intrinsics`.
 * Everything else the call writes (dense gradients, hook tensors, controller accumulators) is bit-identical to
 * gsb200_backward_lens's, whichever camera gradients are on.  NULL pose and NULL intrinsics: exactly
 * gsb200_backward_lens_grad, with the same kernels.  Otherwise, before any CUDA call: the lens checks of
 * gsb200_forward_lens, and those of gsb200_backward_lens_grad (lens_grad), gsb200_backward_pose (pose) and
 * gsb200_backward_calib (intrinsics); GSB_EINVAL for a NULL or pinhole lens; GSB_EUNSUPPORTED for GSB_FLAG_COMPACT_GRADS or
 * num_objects > GSB_POSE_MAX_OBJECTS.  An image-only loss works with either loop-A kernel; the other terms keep their
 * requirement of GSB_FLAG_BACKWARD_TRANSPOSED. */
int gsb200_backward_lens_calib(const GsbBackwardArgs *args, const float *grad_rasterized_depth, const float *rasterized_depth,
                               const float *grad_pixel_accumulated_alpha, const GsbExtraFeatureArgs *ext,
                               const GsbLensArgs *lens, const GsbLensGradArgs *lens_grad, /* or NULL */
                               const GsbPoseGradArgs *pose,                               /* or NULL */
                               const GsbIntrinsicsGradArgs *intrinsics);                  /* or NULL */

/* Rolling shutter (an extension: the reference projects every point with one global-shutter pose).  A view carries a motion
 * m = (v, w) (float32 x 6): the apparent motion of the scene in the camera frame over one full readout, top row to bottom
 * row; v in scene units, w in radians.  The view's pose (q, t) is the pose at mid-readout.  With pc0 = W xyz + tw the camera-
 * frame point of today and the row time tau in [-1/2, 1/2] (0 at the centre row):
 *   pc(tau) = Rd(tau) pc0 + tau v,   Rd(tau) = exp(tau [w]x)   (Rodrigues; a series below |tau w|^2 = 0.01, so w = 0 is I)
 *   row(p) = clamp(v_pix(p) / H - 1/2, -1/2, 1/2)   (v_pix: the row coordinate of p, through the lens if there is one;
 *                                                    a NaN row clamps to -1/2)
 *   tau_0 = 0,  tau_(k+1) = row(pc(tau_k)),  k < GSB_RS_ITERATIONS;  the point is rendered at pc(tau_3).
 * Everything downstream uses pc(tau_3) and W_eff = Rd(tau_3) W: the near / far / border tests, the lens r_max test, (u, v),
 * the depth and sort key, J and Sigma' = J W_eff Sigma W_eff^T J^T.  The SH view direction keeps the mid-readout camera centre.
 * With m = 0, Rd = I and tau v = 0 exactly, so the rolling-shutter calls reproduce the global-shutter calls bit for bit.
 * Gradients: tau is detached (like J, rescale and the SH direction); the point gradients flow through W_eff and pc(tau), and
 * the per-point backward reads tau back from `row_time` instead of solving for it again.  The motion gradient (opt-in,
 * GsbRollingShutterGradArgs), with gp = dL/dpc and [B0; B1] the rows of G (J W_eff) Sigma:
 *   dL/dv = sum_i tau_i gp_i
 *   dL/dRd_i = gp_i pc0_i^T + 2 J^T [B0; B1] W^T   (the full 2x3 J: with a lens it is not sparse)
 *   dL/dw = sum_i tau_i J_r(tau_i w)^T a(Rd_i^T dL/dRd_i),  a(A) = (A32 - A23, A13 - A31, A21 - A12)
 * summed over every in-camera point of every object (rolling_shutter_grad in csrc/common.cuh).  Every loss term that reaches
 * the accumulator rows contributes (image, depth with its direct dL/dz, alpha, features).  The sum is deterministic: the
 * per-point kernel runs on min(ceil(N/128), GSB_RS_GRAD_PARTIAL_BLOCKS) CTAs, each writes its sums to `temp`, and a second
 * kernel adds them in block order -- no float atomics. */
#define GSB_RS_ITERATIONS 3
#define GSB_RS_GRAD_PARTIAL_BLOCKS 2048
typedef struct GsbRollingShutterArgs {
    float motion[6];  /* v (3), w (3) */
    float *row_time;  /* (N,) float32, 4-byte aligned: written by the forward (tau_3 in camera, 0 outside the frustum), read
                       * by the backward of the same frame */
} GsbRollingShutterArgs;
typedef struct GsbRollingShutterGradArgs {
    float *grad_motion; /* (6,) out, dL/dv then dL/dw */
    void *temp;         /* gsb200_rolling_shutter_grad_temp_bytes() bytes, 16-byte aligned */
} GsbRollingShutterGradArgs;
/* GSB_RS_GRAD_PARTIAL_BLOCKS * 6 floats */
int64_t gsb200_rolling_shutter_grad_temp_bytes(void);
/* gsb200_forward_lens through the rolling shutter of `rs`.  NULL rs: exactly gsb200_forward_lens.  Before any CUDA call: the
 * lens checks of gsb200_forward_lens; GSB_EINVAL for a non-finite motion or a NULL or misaligned row_time. */
int gsb200_forward_rolling_shutter(const GsbForwardArgs *args, const GsbExtraFeatureArgs *ext, const GsbLensArgs *lens,
                                   const GsbRollingShutterArgs *rs);  /* lens, rs or NULL */
/* gsb200_backward_lens of a frame rendered by gsb200_forward_rolling_shutter with the same lens and rs.  NULL rs: exactly
 * gsb200_backward_lens.  NULL rs_grad: no motion gradient; every other output is bit-identical to the call with rs_grad.
 * Before any CUDA call: the checks of gsb200_forward_rolling_shutter; GSB_EINVAL for an rs_grad without rs, a NULL output or
 * temp pointer, an output that is not 4-byte aligned or a temp that is not 16-byte aligned; GSB_EUNSUPPORTED for
 * GSB_FLAG_COMPACT_GRADS.  An image-only loss works with either loop-A kernel; the other terms keep their requirement of
 * GSB_FLAG_BACKWARD_TRANSPOSED. */
int gsb200_backward_rolling_shutter(const GsbBackwardArgs *args, const float *grad_rasterized_depth,
                                    const float *rasterized_depth, const float *grad_pixel_accumulated_alpha,
                                    const GsbExtraFeatureArgs *ext, const GsbLensArgs *lens, const GsbRollingShutterArgs *rs,
                                    const GsbRollingShutterGradArgs *rs_grad);  /* lens, rs, rs_grad or NULL */

/* Motion blur (an extension: the reference renders every view as if the shutter were instantaneous).  A view may carry an
 * exposure motion m_b = (v, w) (float32 x 6): the apparent motion of the scene in the camera frame over the whole exposure,
 * in the convention of GsbRollingShutterArgs::motion; the view's pose is the pose at mid-exposure.  With pc the camera-frame
 * point as rendered without blur (with a rolling shutter: pc(tau_3), and W is W_eff) and Jp = d(u, v)/d pc the full position
 * Jacobian (full K, and the lens D when there is one):
 *   d = Jp (v + w x pc)                  the screen displacement of the splat centre over the exposure
 *   B = d d^T / 12                       the second moment of a uniform sweep t in [-1/2, 1/2]
 *   conic = (Sigma_d + B)^-1,  Sigma_d = Sigma' + 0.3 I
 *   rescale slot = rescale c_b,  rescale = sqrt(det Sigma' / det Sigma_d) (detached),  c_b = sqrt(det Sigma_d / det(Sigma_d + B))
 *   radius (and the tile square) from Sigma' + B; the reach test runs on the blurred conic
 * c_b keeps each splat's integrated weight over the sweep.  m_b = 0 takes the un-blurred arithmetic: records, keys, images and
 * every gradient are those of the call without blur, bit for bit.  The model replaces the box-shaped streak by a Gaussian of
 * equal variance, linearises the screen trajectory at mid-exposure and composites time-averaged splats.
 * Only +-m_b is observable (B depends on d d^T alone), and dB/dm_b = 0 at m_b = 0: refining m_b needs a non-zero start.
 * Gradients: d is detached with respect to the point (like J, tau and rescale).  With G = dL/dSigma' of the blend and
 * G_a = glogit / fl(1 - o) (the 3D filter's recovery of sum dL/dalpha alpha; dropped where fl(1 - o) = 0):
 *   dL/dSigma' = G + G_a/2 (Sigma_d^-1 - (Sigma_d + B)^-1)
 *   dL/dd = G d / 6 - G_a/12 (Sigma_d + B)^-1 d,   g = Jp^T dL/dd
 *   dL/dv = sum_i g_i,   dL/dw = sum_i pc_i x g_i
 * summed over every in-camera point of every object (GsbMotionBlurGradArgs; every loss term that reaches the accumulator rows
 * contributes).  The sum is deterministic as the rolling shutter's: min(ceil(N/128), GSB_RS_GRAD_PARTIAL_BLOCKS) per-CTA rows
 * in `temp`, added in block order by a second kernel.  Not implemented with the 3D filter, the rolling-shutter motion
 * gradient, pose / intrinsics / lens-coefficient gradients or the compact rows of the view-parallel exchange. */
typedef struct GsbMotionBlurArgs {
    float motion[6];  /* v (3), w (3) over the whole exposure */
} GsbMotionBlurArgs;
typedef struct GsbMotionBlurGradArgs {
    float *grad_motion; /* (6,) out, dL/dv then dL/dw */
    void *temp;         /* gsb200_motion_blur_grad_temp_bytes() bytes, 16-byte aligned */
} GsbMotionBlurGradArgs;
/* GSB_RS_GRAD_PARTIAL_BLOCKS * 6 floats */
int64_t gsb200_motion_blur_grad_temp_bytes(void);
/* sizeof(GsbMotionBlurArgs), sizeof(GsbMotionBlurGradArgs) (a call of their own, like gsb200_abi_sizes_mcmc) */
void gsb200_abi_sizes_motion_blur(int64_t *out2);
/* gsb200_forward_rolling_shutter with the exposure motion of `blur`.  NULL blur: exactly gsb200_forward_rolling_shutter.
 * Before any CUDA call: the checks of gsb200_forward_rolling_shutter; GSB_EINVAL for a non-finite motion. */
int gsb200_forward_motion_blur(const GsbForwardArgs *args, const GsbExtraFeatureArgs *ext, const GsbLensArgs *lens,
                               const GsbRollingShutterArgs *rs, const GsbMotionBlurArgs *blur);  /* lens, rs, blur or NULL */
/* gsb200_backward_rolling_shutter (without the rolling-shutter motion gradient) of a frame rendered by
 * gsb200_forward_motion_blur with the same lens, rs and blur.  NULL blur: exactly gsb200_backward_rolling_shutter(..., NULL).
 * NULL blur_grad: no motion gradient; every other output is bit-identical to the call with blur_grad.  Before any CUDA call:
 * the checks of gsb200_forward_motion_blur; GSB_EINVAL for a blur_grad without blur, a NULL output or temp pointer, an output
 * that is not 4-byte aligned or a temp that is not 16-byte aligned; GSB_EUNSUPPORTED for GSB_FLAG_COMPACT_GRADS.  An
 * image-only loss works with either loop-A kernel; the other terms keep their requirement of GSB_FLAG_BACKWARD_TRANSPOSED. */
int gsb200_backward_motion_blur(const GsbBackwardArgs *args, const float *grad_rasterized_depth, const float *rasterized_depth,
                                const float *grad_pixel_accumulated_alpha, const GsbExtraFeatureArgs *ext,
                                const GsbLensArgs *lens, const GsbRollingShutterArgs *rs, const GsbMotionBlurArgs *blur,
                                const GsbMotionBlurGradArgs *blur_grad);  /* lens, rs, blur, blur_grad or NULL */

/* Depth of field (an extension: the reference renders through an ideal pinhole).  A view may carry a thin lens (a, rho)
 * (float32 x 2): a the aperture diameter in scene units, rho = 1 / focus distance in 1/scene units (0: focused at infinity).
 * Both live on the normalised image plane, so downsampling, crop and autoscale leave them unchanged.  With pc the rendered
 * camera-frame point (pc(tau_3) with a rolling shutter), z = pc.z and M = K[:2,:2] (K[:2,:2] D with a lens, the 2x2 factor of
 * Jp above):
 *   beta = a^2 (rho - 1/z)^2 / 16        the per-axis variance of a uniform disk of diameter a |rho - 1/z| on the normalised plane
 *   B_d = beta M M^T,  B = B_m + B_d     (B_m the motion blur's d d^T / 12 when the view also has one, else 0)
 * and the conic, rescale slot (c_b), radius, tile square and reach test follow from Sigma_d + B as for the motion blur.  The
 * model is exact at the level of the covariance: an aperture sample s moves the camera centre by s and, to keep the focal
 * plane fixed, the principal point by M s rho, so a point moves by M s (rho - 1/z) and its covariance over the disk is B_d.
 * The blur diameter in pixels is a f_px |rho - 1/z|.  It approximates the disk by a Gaussian of equal variance, composites
 * defocused splats instead of averaging composited frames (no partial occlusion at depth edges) and, with a lens, maps the
 * disk through the lens Jacobian at the point.  a = 0 takes the arithmetic without defocus: records, keys, images and every
 * gradient are those of gsb200_forward_motion_blur / gsb200_backward_motion_blur, bit for bit.
 * Only |a| is observable, and both parameter gradients vanish at a = 0: refinement needs a non-zero start.  rho is
 * identifiable only from a view spanning a range of depths: points in front of and behind the focal plane blur alike.
 * Gradients: beta is detached with respect to the point (like J and d).  With G and G_a as for the motion blur:
 *   G_B = G - G_a/2 (Sigma_d + B)^-1,   dL/dbeta = <G_B, M M^T>
 *   dL/da = sum_i dL/dbeta_i a (rho - 1/z_i)^2 / 8,   dL/drho = sum_i dL/dbeta_i a^2 (rho - 1/z_i) / 8
 * over every in-camera point (GsbDefocusGradArgs), deterministic as the motion blur's: the per-CTA rows in `temp` and the
 * block-order finishing kernel.  dL/dSigma' has the motion blur's form with this B.  Not implemented with the 3D filter,
 * camera-parameter gradients (pose, intrinsics, lens coefficients, rolling-shutter or exposure motion) or the compact rows of
 * the view-parallel exchange. */
typedef struct GsbDefocusArgs {
    float aperture;       /* a, scene units */
    float inverse_focus;  /* rho = 1 / focus distance */
} GsbDefocusArgs;
typedef struct GsbDefocusGradArgs {
    float *grad; /* (2,) out, dL/da, dL/drho */
    void *temp;  /* gsb200_defocus_grad_temp_bytes() bytes, 16-byte aligned */
} GsbDefocusGradArgs;
/* (GSB_RS_GRAD_PARTIAL_BLOCKS + 1) * 6 floats: the per-CTA rows and the finished row */
int64_t gsb200_defocus_grad_temp_bytes(void);
/* sizeof(GsbDefocusArgs), sizeof(GsbDefocusGradArgs) (a call of their own, like gsb200_abi_sizes_motion_blur) */
void gsb200_abi_sizes_defocus(int64_t *out2);
/* gsb200_forward_motion_blur with the thin lens of `defocus`.  NULL defocus: exactly gsb200_forward_motion_blur.  Before any
 * CUDA call: the checks of gsb200_forward_motion_blur; GSB_EINVAL for a non-finite a or rho. */
int gsb200_forward_defocus(const GsbForwardArgs *args, const GsbExtraFeatureArgs *ext, const GsbLensArgs *lens,
                           const GsbRollingShutterArgs *rs, const GsbMotionBlurArgs *blur,
                           const GsbDefocusArgs *defocus);  /* lens, rs, blur, defocus or NULL */
/* gsb200_backward_motion_blur (without the exposure-motion gradient) of a frame rendered by gsb200_forward_defocus with the
 * same lens, rs, blur and defocus.  NULL defocus: exactly gsb200_backward_motion_blur(..., blur, NULL).  NULL defocus_grad: no
 * (a, rho) gradient; every other output is bit-identical to the call with defocus_grad.  Before any CUDA call: the checks of
 * gsb200_forward_defocus; GSB_EINVAL for a defocus_grad without defocus, a NULL output or temp pointer, an output that is not
 * 4-byte aligned or a temp that is not 16-byte aligned; GSB_EUNSUPPORTED for GSB_FLAG_COMPACT_GRADS. */
int gsb200_backward_defocus(const GsbBackwardArgs *args, const float *grad_rasterized_depth, const float *rasterized_depth,
                            const float *grad_pixel_accumulated_alpha, const GsbExtraFeatureArgs *ext, const GsbLensArgs *lens,
                            const GsbRollingShutterArgs *rs, const GsbMotionBlurArgs *blur, const GsbDefocusArgs *defocus,
                            const GsbDefocusGradArgs *defocus_grad);  /* lens, rs, blur, defocus, defocus_grad or NULL */

int gsb200_expand_view_gradients(const GsbExpandArgs *args);

/* The two collectives of the compact exchange as ONE hand-written kernel over NVSwitch multicast memory (NVLS; csrc/exchange.cu):
 * a two-shot all-reduce of grad_sum (multimem.ld_reduce of this rank's 1/R of the rows, multimem.st of the sums to all ranks)
 * and an all-gather of the per-view blocks (multimem.st of this rank's block into slot `rank` on all ranks).  The buffers must
 * live in one symmetric allocation mapped to a multicast address (torch.distributed._symmetric_memory); the caller brackets the
 * call with two cross-rank barriers on the same stream: all ranks' compact rows written before, all multicast stores landed
 * after (parallel.MulticastViewParallelExchange).  The alternative to ncclAllReduce + ncclAllGather of the NCCL path. */
typedef struct GsbMultimemExchangeArgs {
    int64_t num_points;
    int32_t num_objects, rank, world_size;
    int32_t num_blocks;          /* CTAs to launch; 0 = 2 per SM */
    int32_t phases;              /* 0 or 3 = both; 1 = only the all-gather push of this rank's block (needs no barrier in front if
                                    the caller alternates the blocks buffer with the step parity); 2 = only the all-reduce */
    int32_t reserved;
    float *multicast_grad_sum;   /* multicast address of the (N,12) rows */
    float *multicast_blocks;     /* multicast address of the (world_size, block_stride) blocks */
    const float *local_block;    /* this rank's own block [3N | 3 n_obj], local address */
    int64_t block_stride;        /* floats, multiple of 4, >= 3N + 3 n_obj */
    void *stream;
} GsbMultimemExchangeArgs;
int gsb200_exchange_multimem(const GsbMultimemExchangeArgs *args);

/* One WHOLE training iteration of the reference loop (GaussianPointTrainer.py:138-180) enqueued by one call, without any host
 * interaction: forward (gsb200_forward) -> clamp + L1 + D-SSIM loss and its gradient (gsb200_image_loss, LossFunction.py:20-38
 * without the optional scale regulariser) -> backward (gsb200_backward, with the controller accumulators if set) -> Adam on the
 * features and on the positions (gsb200_adam_step, GaussianPointTrainer.py:126-129, 176-177).  The scene tensors of `forward`
 * are updated in place.  `backward` must describe the same frame (same scene / workspace / sizes), with
 * grad_rasterized_image = the (H,W,3) buffer the loss gradient is written to and accum_rows >= num_points (the number of
 * in-camera points is not known on the host).  If the frame needs more (tile, splat) pairs than forward.key_capacity the
 * device-side overflow counter makes the accumulator update and both Adam steps no-ops; the host sees it in
 * forward.host_counters[2] (async copy, never waited on here) and must repeat the iteration with a larger capacity. */
typedef struct GsbTrainStepArgs {
    GsbForwardArgs forward;
    GsbBackwardArgs backward;
    const float *ground_truth_image; /* (3,H,W) as the dataset yields it */
    float lambda_value;              /* LossFunction.py:23 */
    float *loss_out3;                /* device: {loss, L1, 1 - SSIM} */
    void *loss_temp;                 /* gsb200_image_loss_temp_bytes(H, W), first 16 bytes zero before the first use */
    int64_t loss_temp_bytes;
    float *feature_exp_avg, *feature_exp_avg_sq;   /* (N,56) Adam state, zero before the first step */
    float *position_exp_avg, *position_exp_avg_sq; /* (N,3) */
    double feature_learning_rate, position_learning_rate, beta1, beta2, eps;
    int32_t step;                    /* 1-based Adam step count */
} GsbTrainStepArgs;
int gsb200_train_step(const GsbTrainStepArgs *args);

/* Depth, mask and background terms of the fused train step (an extension: the reference trains on the image alone).  For a
 * view with I the rasterised image, S = pixel_accumulated_alpha, D = the rendered depth:
 *   background (if set):  the image loss runs on I' = I + (1 - S) bg; with a mask target the ground truth is composited
 *                         too, gt' = gt m + (1 - m) bg (without one it is taken to be on bg already);
 *   mask term:            mask_weight * mean |S - m|;
 *   depth term:           depth_weight * sum_valid |D - d*| / max(n_valid, 1), a pixel valid when d* is finite and > 0
 *                         (0 or NaN = no measurement); d* in point-cloud units along the optical axis, like D.
 * total = image loss + mask term + depth term.  The gradients w.r.t. S and D are written to the caller's buffers and fed to
 * the backward (gsb200_backward_aux). */
typedef struct GsbSupervisionArgs {
    const float *depth_target;    /* (H,W) f32 or NULL */
    const float *mask_target;     /* (H,W) f32 in [0,1] or NULL */
    const float *background;      /* device float[3] or NULL (black: no compositing) */
    float depth_weight, mask_weight; /* >= 0, finite; 0 = term off */
    float *grad_depth;            /* (H,W) out: dL/dD (depth term) */
    float *grad_pixel_accumulated_alpha; /* (H,W) out: dL/dS (mask term or background) */
    float *loss_out3;             /* device: {total, mask term, depth term} */
    void *temp;                   /* gsb200_supervision_temp_bytes(H, W), 16-byte aligned, first 16 bytes zero before first use */
    int64_t temp_bytes;
} GsbSupervisionArgs;
int64_t gsb200_supervision_temp_bytes(int32_t camera_height, int32_t camera_width);
/* gsb200_train_step with the supervision terms: forward -> pre-pass (composite, sums) -> image loss on (I', gt') ->
 * post-pass (dL/dS, dL/dD, losses) -> backward with the depth and alpha gradients (skipped on overflow like the rest) ->
 * both Adam steps.  NULL supervision, or every term off: exactly gsb200_train_step.  GSB_EINVAL, before any CUDA call, for a
 * negative or non-finite weight, a weight > 0 without its target or gradient output, a background without the alpha
 * gradient output, or a temp that is too small or not 16-byte aligned; GSB_EUNSUPPORTED without
 * GSB_FLAG_BACKWARD_TRANSPOSED.  Deterministic: fixed grids and summation orders. */
int gsb200_train_step_aux(const GsbTrainStepArgs *args, const GsbSupervisionArgs *supervision);

/* Feature term of the fused train step (an extension): a loss on the per-Gaussian feature map F = features.rasterized
 * (H,W,C) that gsb200_forward_ext renders, back-propagated by gsb200_backward_ext, and an Adam step on the (N,C) features.
 *   GSB_FEATURE_LOSS_CROSS_ENTROPY (semantic labels, C >= 2): labels (H,W) int32, a pixel labelled when 0 <= label < C;
 *     weight * sum_labelled CE(softmax(F_p), label_p) / max(n_labelled, 1), with a max-subtracted log-sum-exp;
 *   GSB_FEATURE_LOSS_L2 (distilled feature maps): target (H,W,C) f32, a pixel supervised when all C values are finite (NaN =
 *     no target); weight * sum_supervised sum_c (F_pc - T_pc)^2 / max(n_supervised * C, 1).
 * An unsupervised pixel gets a zero gradient; a frame without one supervised pixel has term 0. */
#define GSB_FEATURE_LOSS_CROSS_ENTROPY 1
#define GSB_FEATURE_LOSS_L2 2
typedef struct GsbFeatureTrainArgs {
    GsbExtraFeatureArgs features; /* features (N,C): updated in place by Adam; rasterized (H,W,C): the forward's feature map;
                                     grad_rasterized (H,W,C): written by the loss (dL/dF); grad_features (N,C): dL/df */
    int32_t loss_kind;            /* GSB_FEATURE_LOSS_* */
    float weight;                 /* > 0, finite */
    const int32_t *labels;        /* (H,W) cross entropy (not read for l2) */
    const float *target;          /* (H,W,C) l2 (not read for cross entropy) */
    float *loss_out2;             /* device: {feature term, n_supervised} */
    void *temp;                   /* gsb200_feature_loss_temp_bytes(H, W), 16-byte aligned, first 16 bytes zero before first use */
    int64_t temp_bytes;
    float *exp_avg, *exp_avg_sq;  /* (N,C) Adam state of the features, zero before the first step, 16-byte aligned */
    double learning_rate;         /* Adam of the features; betas, eps and step are the train step's */
} GsbFeatureTrainArgs;
int64_t gsb200_feature_loss_temp_bytes(int32_t camera_height, int32_t camera_width);
/* gsb200_train_step_aux with the feature term: gsb200_forward_ext -> the supervision pre-pass, image loss and post-pass
 * (unchanged) -> feature loss (pass 1: sums, pass 2: dL/dF and loss_out2) -> gsb200_backward_ext with the depth, alpha and
 * feature gradients -> Adam on the 56 columns, on xyz and on the features, all three skipped on the device after a
 * key-capacity overflow.  NULL features: exactly gsb200_train_step_aux (which is this call with NULL).  Before any CUDA call:
 * GSB_EINVAL for channels outside 1..16, an unknown kind, cross entropy with C < 2, a weight that is not finite or not > 0,
 * a NULL target, map, gradient, moment or output pointer, a temp that is too small or not 16-byte aligned, or features,
 * grad_features or moments that are not 16-byte aligned; GSB_EUNSUPPORTED without GSB_FLAG_BACKWARD_TRANSPOSED or with
 * GSB_FLAG_COMPACT_GRADS.  Deterministic: fixed grids and summation orders. */
int gsb200_train_step_ext(const GsbTrainStepArgs *args, const GsbSupervisionArgs *supervision,
                          const GsbFeatureTrainArgs *features);

/* Per-view appearance compensation (an extension): a bilateral grid (Wang et al., "Bilateral Guided Radiance Field
 * Processing", SIGGRAPH 2024) of one view, G with shape (12, Gz, Gy, Gx), float32, contiguous: a 3x4 affine [A | b] (row-major)
 * per node, Gx / Gy nodes across the image width / height, Gz over luminance; 1 <= Gx, Gy <= 64, 1 <= Gz <= 16.  For an
 * image I (H,W,3), at pixel (px, py) with colour c:
 *   gx = px (Gx-1) / max(W-1, 1),  gy = py (Gy-1) / max(H-1, 1)
 *   lum = clamp(0.299 c_r + 0.587 c_g + 0.114 c_b, 0, 1),  gz = lum (Gz-1)
 *   [A | b] = trilinear interpolation of G at (gx, gy, gz), the lower corner index clamped to n-2;  out = A c + b
 * -- exactly F.grid_sample(G[None], (x, y, 2 lum - 1) in [-1, 1], mode="bilinear", align_corners=True,
 * padding_mode="border").  The identity grid (A = I, b = 0) reproduces the image.  The backward gives dL/dG and dL/dc, the
 * latter through A and, where 0 < lum < 1, through lum (the slope of the interpolation along z times (Gz-1) times
 * (0.299, 0.587, 0.114)).  The TV prior is tv(G) = sum over the x, y and z axes of mean((G[i+1] - G[i])^2); an axis with one
 * node contributes 0.  Deterministic: dL/dG is summed per grid cell in a fixed order, with no float atomics. */
#define GSB_BILATERAL_GRID_MAX_XY 64
#define GSB_BILATERAL_GRID_MAX_Z 16
/* bytes of the backward's temp (per-CTA partial sums of dL/dG); 0 for a shape outside the limits */
int64_t gsb200_bilateral_grid_temp_bytes(int32_t camera_height, int32_t camera_width, int32_t grid_x, int32_t grid_y,
                                         int32_t grid_z);
/* image_out (H,W,3) = the slice of `grid` applied to image (H,W,3).  GSB_EINVAL, before any CUDA call, for a shape outside
 * the limits or a NULL or not 4-byte aligned pointer. */
int gsb200_bilateral_grid_forward(const float *image, const float *grid, int32_t camera_height, int32_t camera_width,
                                  int32_t grid_x, int32_t grid_y, int32_t grid_z, float *image_out, void *stream);
/* From dL/dout (H,W,3): grad_image (H,W,3) = dL/dimage (it may alias grad_image_out: each pixel is read before it is
 * written) and grad_grid (12,Gz,Gy,Gx) = dL/dG (overwritten).  GSB_EINVAL, before any CUDA call, for a shape outside the
 * limits, a NULL or not 4-byte aligned pointer, or a temp that is NULL, not 16-byte aligned or smaller than
 * gsb200_bilateral_grid_temp_bytes. */
int gsb200_bilateral_grid_backward(const float *image, const float *grid, int32_t camera_height, int32_t camera_width,
                                   int32_t grid_x, int32_t grid_y, int32_t grid_z, const float *grad_image_out,
                                   float *grad_image, float *grad_grid, void *temp, int64_t temp_bytes, void *stream);

/* The appearance grid of the view a fused train step trains on. */
typedef struct GsbAppearanceArgs {
    float *grid;                  /* (12,Gz,Gy,Gx) this view's grid, updated in place by its Adam step */
    float *grad_grid;             /* (12,Gz,Gy,Gx) out: dL/dG (slice and TV) */
    int32_t grid_x, grid_y, grid_z;
    float tv_weight;              /* >= 0, finite */
    float *exp_avg, *exp_avg_sq;  /* (12,Gz,Gy,Gx) this view's Adam moments, zero before its first step */
    double learning_rate;         /* >= 0, finite; betas and eps are the train step's */
    int32_t step;                 /* this view's own 1-based Adam step count */
    float *image;                 /* (H,W,3) scratch: the sliced image I'' the image loss reads */
    void *temp;                   /* gsb200_bilateral_grid_temp_bytes(H, W, Gx, Gy, Gz) bytes, 16-byte aligned */
    int64_t temp_bytes;
    float *loss_out1;             /* device: {tv_weight * tv(G)} */
} GsbAppearanceArgs;
/* gsb200_train_step_ext with the view's appearance grid: forward -> supervision pre-pass -> slice I'' = grid(I') of the image
 * the loss would read (I' = I + (1 - S) bg with a background, else I) -> image loss on I'' -> slice backward (dL/dG, and
 * dL/dI' in place over the image-loss gradient) -> TV (added into dL/dG, loss_out1) -> supervision post-pass (reads dL/dI')
 * -> feature loss -> backward -> the Adam steps, then Adam on the grid; all of them skipped on the device after a
 * key-capacity overflow.  The depth, mask and feature terms do not see the grid.  NULL appearance: exactly
 * gsb200_train_step_ext.  GSB_EINVAL, before any CUDA call, for a shape outside the limits, a NULL or not 16-byte aligned
 * grid, gradient, moment, image or temp pointer, a NULL loss_out1, a temp smaller than gsb200_bilateral_grid_temp_bytes,
 * step < 1, or a TV weight or learning rate that is negative or not finite.  Deterministic. */
int gsb200_train_step_appearance(const GsbTrainStepArgs *args, const GsbSupervisionArgs *supervision,
                                 const GsbFeatureTrainArgs *features, const GsbAppearanceArgs *appearance);

/* MCMC densification (an extension; Kheradmand et al., "3D Gaussian Splatting as Markov Chain Monte Carlo", NeurIPS 2024):
 * the per-iteration regularisers and position noise, and the relocation arithmetic of a refinement.  Row layout as
 * everywhere: features[0:4] = q (xyzw), [4:7] = log-scale s, [7] = opacity logit; o = sigmoid(logit), scale = exp(s),
 * Sigma = R(q / |q|) diag(exp(2 s)) R^T.  A row is valid when point_invalid_mask == 0; n_v = the number of valid rows (the
 * host knows it: it changes only at a refinement).
 *   Regularisers:  R = lambda_o sum_valid o_i / n_v + lambda_s sum_valid sum_j exp(s_ij) / (3 n_v)
 *     dR/dlogit_i = lambda_o o_i (1 - o_i) / n_v,  dR/ds_ij = lambda_s exp(s_ij) / (3 n_v); invalid rows get nothing.  Plain
 *     derivatives: the rasteriser's gradient factors (GsbBackwardArgs::grad_*_factor) do not apply to them.  n_v = 0: R = 0.
 *   Position noise, after the optimiser step of iteration t, for every valid row i:
 *     xyz_i += Sigma_i eps_i noise_scale g(o_i),  g(o) = 1 / (1 + exp(-gate_k ((1 - o) - (1 - min_opacity))))
 *     (noise_scale = noise_lr * the position learning rate of the step; the paper: gate_k = 100, min_opacity = 0.005).
 *     eps_i in R^3 is a pure function of (seed, t, i): x[0..3] = Philox4x32-10 (Salmon et al., SC 2011; multipliers
 *     0xD2511F53, 0xCD9E8D57, key increments 0x9E3779B9, 0xBB67AE85) with key = {seed low, seed high 32 bits} and counter =
 *     {i low, i high, t low, t high};  u_k = ((x[k] >> 9) + 0.5) 2^-23, exact in float32 and never 0 or 1 (a 24-bit mantissa
 *     cannot hold (x >> 8) + 0.5);  Box-Muller:  eps = (r0 cos(2 pi u_1), r0 sin(2 pi u_1), r1 cos(2 pi u_3)),
 *     r0 = sqrt(-2 ln u_0), r1 = sqrt(-2 ln u_2).  No state is kept: two calls with equal arguments are bit-identical.
 *   Relocation (the paper's eq. 9), for a source that ends up as n copies (times drawn + 1, clamped to GSB_MCMC_N_MAX):
 *     o_new = 1 - (1 - o)^(1/n),  D = sum_{i=1..n} sum_{k=0..i-1} C(i-1, k) (-1)^k o_new^(k+1) / sqrt(k+1),
 *     s_new = s + log(o / D),  logit_new = logit(clamp(o_new, min_opacity, 1 - 1e-7));  evaluated in double (the sum
 *     alternates); n = 1 is the identity to rounding (D = o). */
#define GSB_MCMC_N_MAX 51
/* bytes of the regulariser's temp (a ticket and per-CTA partial sums) */
int64_t gsb200_mcmc_temp_bytes(void);
/* Adds dR/dfeatures into columns 4..7 of grad_features (N,56) -- the gradient the backward has just written -- and writes
 * terms_out2 = {opacity term, scale term} of R (device).  The sums are taken in double in a fixed order: bit-reproducible.
 * temp: gsb200_mcmc_temp_bytes() bytes, its first 16 bytes zero before the first use (the call leaves them ready for the next
 * one).  GSB_EINVAL, before any CUDA call, for num_points < 0, num_valid outside [0, num_points], a weight that is negative
 * or not finite, or a NULL or not 16-byte aligned features, grad_features or temp pointer, a NULL mask or terms_out2. */
int gsb200_mcmc_regulariser(const float *pointcloud_features, const int8_t *point_invalid_mask, float *grad_features,
                            int64_t num_points, int64_t num_valid, float lambda_opacity, float lambda_scale,
                            float *terms_out2, void *temp, void *stream);
/* The position noise of iteration `step` on the valid rows of pointcloud (N,3), in place.  GSB_EINVAL, before any CUDA call,
 * for num_points < 0, step < 0, a noise_scale, gate_k or min_opacity that is negative or not finite, a NULL pointer, a
 * pointcloud that is not 4-byte aligned or features that are not 16-byte aligned. */
int gsb200_mcmc_noise(float *pointcloud, const float *pointcloud_features, const int8_t *point_invalid_mask,
                      int64_t num_points, float noise_scale, float gate_k, float min_opacity, uint64_t seed, int64_t step,
                      void *stream);
/* One relocation: first every drawn source row gets its new logit and log-scales from its draw count (in place) and its Adam
 * moments zeroed; then, in stream order, every destination row becomes a copy of its source's updated row (xyz, the 56
 * features, the object id, the extra-feature row when present), its mask byte is cleared and its moments are zeroed.  The
 * caller guarantees: source ids unique, destination ids unique and disjoint from the source ids (no atomics are used).  A row
 * id outside [0, num_points) is skipped on the device. */
typedef struct GsbMcmcRelocateArgs {
    int64_t num_points;
    int64_t num_sources;
    const int32_t *source_ids;        /* (num_sources,) rows that were drawn at least once */
    const int32_t *source_counts;     /* (num_sources,) times drawn; the row ends up as count + 1 copies */
    int64_t num_destinations;
    const int32_t *destination_ids;   /* (num_destinations,) rows that are overwritten */
    const int32_t *destination_sources; /* (num_destinations,) the row each one copies */
    float *pointcloud;                /* (N,3) */
    float *pointcloud_features;       /* (N,56), 16-byte aligned */
    int8_t *point_invalid_mask;       /* (N,) */
    int32_t *point_object_id;         /* (N,) */
    float *extra_features;            /* (N,C) or NULL */
    int32_t channels;                 /* C in 1..16 with extra_features */
    float min_opacity;                /* in (0, 1) */
    float *feature_exp_avg, *feature_exp_avg_sq;   /* (N,56) 16-byte aligned, or both NULL */
    float *position_exp_avg, *position_exp_avg_sq; /* (N,3) or both NULL */
    float *extra_exp_avg, *extra_exp_avg_sq;       /* (N,C) or both NULL (need extra_features) */
    void *stream;
} GsbMcmcRelocateArgs;
/* GSB_EINVAL, before any CUDA call, for a NULL args, counts outside [0, num_points], a NULL id array with a non-zero count,
 * a NULL scene tensor, features or feature moments that are not 16-byte aligned, C outside 1..16, a moment pair with one
 * NULL half, extra moments without extra_features, or min_opacity outside (0, 1). */
int gsb200_mcmc_relocate(const GsbMcmcRelocateArgs *args);

/* The MCMC part of a fused train step. */
typedef struct GsbMcmcStepArgs {
    int64_t num_valid;                  /* n_v in [0, num_points] */
    float lambda_opacity, lambda_scale; /* >= 0, finite */
    float noise_scale;                  /* noise_lr * this step's position learning rate; >= 0, finite */
    float gate_k, min_opacity;          /* >= 0, finite */
    uint64_t seed;
    int64_t step;                       /* the iteration t of the noise counter, >= 0 */
    float *terms_out2;                  /* device: {opacity term, scale term} */
    void *temp;                         /* gsb200_mcmc_temp_bytes(), 16-byte aligned, first 16 bytes zero before first use */
} GsbMcmcStepArgs;
/* gsb200_train_step_appearance with the MCMC per-iteration work: ... -> backward -> regulariser (adds into the dense feature
 * gradient, writes terms_out2) -> the Adam steps -> position noise (reads the updated features).  Both new launches are
 * skipped on the device after a key-capacity overflow, like the Adam steps.  NULL mcmc: exactly
 * gsb200_train_step_appearance.  GSB_EINVAL, before any CUDA call, for the rules of gsb200_mcmc_regulariser and
 * gsb200_mcmc_noise on the fields above. */
int gsb200_train_step_mcmc(const GsbTrainStepArgs *args, const GsbSupervisionArgs *supervision,
                           const GsbFeatureTrainArgs *features, const GsbAppearanceArgs *appearance,
                           const GsbMcmcStepArgs *mcmc);

/* 3D smoothing filter (an extension; Yu et al., "Mip-Splatting: Alias-free 3D Gaussian Splatting", CVPR 2024): every row
 * is convolved in world space with an isotropic Gaussian whose std sigma_i >= 0 (scene units) is set by the finest sampling
 * interval of the training views that see it, so that a scene rendered closer, at a larger focal length or at a higher
 * resolution than any training view holds no frequency those views did not constrain.  filter3d is a float32 (N,) array,
 * read-only and never differentiated; a NaN or negative entry is read as 0, invalid rows are never read.  Row layout as
 * everywhere: features[4:7] = s (log-scales), features[7] = logit, o = sigmoid(logit).  With e_j = exp(s_j)^2 and
 * e^_j = e_j + sigma^2:
 *   rendered scale   s^_j = sqrt(e^_j)            (R orthogonal: Sigma^ = R diag(e^) R^T = Sigma + sigma^2 I exactly)
 *   compensation     c = sqrt((e_0/e^_0)(e_1/e^_1)(e_2/e^_2)) in (0, 1]   (a product of ratios: no overflow)
 *   rendered opacity o^ = o c
 * Everything downstream of Sigma uses Sigma^ (J, Sigma', the compensated 0.3 low-pass, the radius, the tile box and the reach
 * filter).  c is folded into the record's rescale slot (r1.y = rescale c) and r1.z keeps the raw o, so the blend's
 * rescale * opacity product is rescale * o^ and no blend kernel changes; sigma = 0 leaves a row exactly as without the
 * filter.  The per-point backward uses s^ in M = R diag(s^) and
 *   dL/ds_j = (sum_l dM_lj R_lj) s^_j (e_j / e^_j) + G_a sigma^2 / e^_j,   dL/dlogit unchanged,
 * where G_a = sum over pixels of dL/dalpha alpha is recovered as glogit / fl(1 - o) with o read from the frame's record; where
 * fl(1 - o) = 0 (logit >~ 17.3) the compensation term of that row is dropped.  The gradient factors apply as without the
 * filter; rescale, J(pc) and the SH direction stay detached.  Not implemented with camera-parameter gradients (pose,
 * intrinsics, lens coefficients, motion) or the compact rows of the view-parallel exchange. */
typedef struct GsbFilter3dArgs {
    const float *filter3d;  /* (N,) sigma_i, 4-byte aligned */
} GsbFilter3dArgs;
/* gsb200_forward_rolling_shutter with the 3D filter.  NULL filter: exactly gsb200_forward_rolling_shutter.  GSB_EINVAL,
 * before any CUDA call, for a NULL or not 4-byte aligned filter3d. */
int gsb200_forward_filter3d(const GsbForwardArgs *args, const GsbExtraFeatureArgs *ext, const GsbLensArgs *lens,
                            const GsbRollingShutterArgs *rs, const GsbFilter3dArgs *filter);
/* gsb200_backward_rolling_shutter without the motion gradient, with the 3D filter the frame was rendered with (the same
 * array).  NULL filter: exactly gsb200_backward_rolling_shutter(..., NULL).  GSB_EINVAL, before any CUDA call, for a NULL or
 * not 4-byte aligned filter3d; GSB_EUNSUPPORTED with GSB_FLAG_COMPACT_GRADS. */
int gsb200_backward_filter3d(const GsbBackwardArgs *args, const float *grad_rasterized_depth, const float *rasterized_depth,
                             const float *grad_pixel_accumulated_alpha, const GsbExtraFeatureArgs *ext, const GsbLensArgs *lens,
                             const GsbRollingShutterArgs *rs, const GsbFilter3dArgs *filter);
/* gsb200_train_step_mcmc with the 3D filter in its forward and backward.  NULL filter: exactly gsb200_train_step_mcmc.
 * GSB_EINVAL, before any CUDA call, for a NULL or not 4-byte aligned filter3d. */
int gsb200_train_step_filter3d(const GsbTrainStepArgs *args, const GsbSupervisionArgs *supervision,
                               const GsbFeatureTrainArgs *features, const GsbAppearanceArgs *appearance,
                               const GsbMcmcStepArgs *mcmc, const GsbFilter3dArgs *filter);
/* The filter from the training views.  For a valid row i and a view v with full-resolution K_v, W_v, H_v and the pose of the
 * row's object in that view, mapped as the rasteriser maps it (the forward's pose kernel):
 *   pc = T x,  (u, v) = (K pc)[:2] / z   (pinhole, float32, the preprocess's operation order)
 *   v sees i  iff  z > near_plane  and  -0.15 W <= u <= 1.15 W  and  -0.15 H <= v <= 1.15 H   (bounds formed in float32)
 *   d_i = min over the views that see i of z / f_v,  f_v = fmaxf(K00, K11)   (a view with f_v <= 0 sees nothing, and
 *   neither does one with a NaN K00 or K11: u or v is then NaN); a row whose object id is outside [0, num_objects) matches
 *   no view
 *   a valid row no view sees gets the largest d of the seen rows; if no row is seen, every row gets 0
 *   filter3d_i = sqrt(variance) d_i  (variance in pixels^2 at the finest view; the paper's value is 0.2);  invalid rows: 0.
 * The paper takes the minimum distance over one focal length; this takes the per-view z / f, which equals it for views of
 * one focal length and is the sampling interval itself when they differ.  Every step is a min or a max: bit-deterministic.
 * The views' pose blocks, K, W and H are staged through shared memory in chunks, so any number of views and objects works.
 * Lens distortion and rolling shutters are not modelled here: callers pass the pinhole K and the mid-readout pose. */
typedef struct GsbFilter3dViewsArgs {
    int64_t num_points;
    const float *pointcloud;            /* (N,3) */
    const int8_t *point_invalid_mask;   /* (N,) */
    const int32_t *point_object_id;     /* (N,) in [0, num_objects) */
    int32_t num_objects;                /* >= 1 */
    int32_t num_views;                  /* >= 1 */
    const float *q_pointcloud_camera;   /* (V, num_objects, 4) xyzw, camera -> pointcloud, as the forward takes them */
    const float *t_pointcloud_camera;   /* (V, num_objects, 3) */
    const float *camera_intrinsics;     /* (V, 3, 3) full resolution */
    const int32_t *camera_size;         /* (V, 2) {W, H}, full resolution */
    float near_plane;                   /* finite, >= 0 */
    float variance;                     /* finite, >= 0 */
    float *filter3d;                    /* (N,) out, 4-byte aligned */
    void *temp;                         /* gsb200_filter3d_temp_bytes(V, num_objects) bytes, 16-byte aligned */
    int64_t temp_bytes;
    void *stream;
} GsbFilter3dViewsArgs;
int64_t gsb200_filter3d_temp_bytes(int32_t num_views, int32_t num_objects);
/* GSB_EINVAL, before any CUDA call, for a NULL args, num_points < 0, num_views < 1, num_objects < 1, a NULL or misaligned
 * pointer, a temp smaller than gsb200_filter3d_temp_bytes, or a near plane or variance that is negative or not finite. */
int gsb200_filter3d_from_views(const GsbFilter3dViewsArgs *args);
/* sizeof(GsbFilter3dArgs), sizeof(GsbFilter3dViewsArgs) */
void gsb200_abi_sizes_filter3d(int64_t *out2);

/* Orthographic (parallel-projection) views (an extension: the reference projects through a pinhole).  Camera frame as
 * everywhere (x right, y down, z forward), pc = W xyz + t:
 *   u = K00 x + K01 y + K02,  v = K10 x + K11 y + K12   (K[:2] (x, y, 1), no divide; K's last row is not read)
 * so fx = K00 and fy = K11 are pixels per scene unit.  Covariance: Sigma' = J W Sigma W^T J^T with J = K[:2,:2] [I2 0], which
 * does not depend on pc: d(u, v)/d pc = J exactly and nothing is detached through J.  The 0.3 low-pass, rescale, 3-sigma radius,
 * bounding box and reach filter are the pinhole's.  In view: near < z < far and (u, v) inside the image plus the boundary tiles,
 * as the pinhole.  The depth is z: sort key, depth output, depth gradient and the hook's point_depth.  SH view direction: the
 * camera's forward axis in the object's frame, row 2 of W, the same for every point (detached, as in every model).
 * Pose and intrinsics gradients follow the pinhole's conventions with this J:
 *   dL/dK[r][c] = sum guv_r (x, y, 1)_c + 2 sum_j B_r[j] W[c][j] (c = 0, 1),  B = G (J W) Sigma;  row 2 of dL/dK is zero.
 * Known limit: a translation along the viewing axis changes only z, so it reaches the image only through the sort order and the
 * depth output; the pose gradient along that axis comes from the depth term alone. */
/* gsb200_forward_ext of an orthographic view, with the 3D smoothing filter of gsb200_forward_filter3d when `filter` is set (or
 * NULL).  Before any CUDA call: the checks of gsb200_forward_filter3d; K is not read back and nothing synchronises. */
int gsb200_forward_ortho(const GsbForwardArgs *args, const GsbExtraFeatureArgs *ext, const GsbFilter3dArgs *filter);
/* gsb200_backward_calib of a frame rendered by gsb200_forward_ortho with the same filter; filter, pose and intrinsics may each be
 * NULL.  Before any CUDA call: GSB_EUNSUPPORTED with GSB_FLAG_COMPACT_GRADS or for a filter together with a pose or intrinsics
 * gradient, and GSB_EINVAL under the rules of gsb200_backward_filter3d and gsb200_backward_calib.  An image-only loss works with
 * either loop-A kernel; the other terms keep their requirement of GSB_FLAG_BACKWARD_TRANSPOSED.  The pose and intrinsics sums
 * are deterministic (per-CTA rows and finishing kernels, as gsb200_backward_calib). */
int gsb200_backward_ortho(const GsbBackwardArgs *args, const float *grad_rasterized_depth, const float *rasterized_depth,
                          const float *grad_pixel_accumulated_alpha, const GsbExtraFeatureArgs *ext,
                          const GsbFilter3dArgs *filter, const GsbPoseGradArgs *pose,
                          const GsbIntrinsicsGradArgs *intrinsics);

/* Per-pixel weights of the image loss (an extension), for images whose views hold transient distractors (people, cars,
 * shadows that are in one photo and not the next).  For the image x (H,W,3) the image loss reads (the sliced image with an
 * appearance grid, the composited one with a background) and its ground truth g (3,H,W), with s (H,W) the static weight
 * (1 everywhere when NULL):
 *   r = (|c0 - g0| + |c1 - g1| + |c2 - g2|) / 3 in float32 in this order, c = clamp(x, 0, 1);  bin = min(floor(4096 r), 4095)
 *   b = the smallest bin with (float)cum(b) >= q (float)n, cum the histogram of the bins of the n pixels with s > 0
 *   raw inlier: bin <= b
 *   3x3 inlier: (float)(raw inliers) >= box_threshold (float)(neighbours), over the in-image 3x3 neighbours with s > 0
 *   patch inlier: every pixel of a 16x16 tile, when (float)(3x3 inliers) >= patch_threshold (float)(pixels) over the
 *                 tile's pixels with s > 0
 *   w = s [3x3 inlier or patch inlier] with the robust mask (RobustNeRF, Sabour et al., CVPR 2023, section 4), else w = s.
 * The image loss runs unchanged on x' = w c + (1 - w) g (no FMA contraction: it rounds like torch), so a pixel of weight 0
 * is its ground truth and adds nothing to either term, and dL/dx = w 1[0 <= x <= 1] dL/dx'.  The normalisation stays over
 * all pixels.  stats_out2 = {inlier fraction sum[w > 0 among s > 0] / n (0 when n = 0), threshold (b + 1) / 4096 (1 without
 * the robust mask)}.  Integer counts only: two calls are bit-identical.  H and W must be multiples of 16. */
typedef struct GsbRobustLossArgs {
    const float *static_weight;   /* (H,W) in [0,1], or NULL: 1 everywhere */
    int32_t robust;               /* 1: the inlier mask of this iteration's residual; 0: w = s */
    float inlier_quantile;        /* q in (0, 1] (robust only) */
    float box_threshold;          /* in [0, 1] (robust only) */
    float patch_threshold;        /* in [0, 1] (robust only) */
    float *weight_out;            /* (H,W) out: w */
    float *composite;             /* (H,W,3) scratch out: x' */
    void *temp;                   /* gsb200_robust_temp_bytes(H, W), 16-byte aligned, zero before the first use */
    int64_t temp_bytes;
    float *stats_out2;            /* device: {inlier fraction, threshold} */
} GsbRobustLossArgs;
/* bytes of the temp; 0 unless H and W are positive multiples of 16 */
int64_t gsb200_robust_temp_bytes(int32_t camera_height, int32_t camera_width);
/* gsb200_image_loss with the weights: robust pre-passes -> image loss on (x', gt) -> dL/dx into grad_rasterized_image.
 * The rules of gsb200_train_step_robust on `robust`, and those of gsb200_image_loss; grad_rasterized_image must not be NULL. */
int gsb200_robust_image_loss(const float *rasterized_image, const float *ground_truth_image, int32_t camera_height,
                             int32_t camera_width, float lambda_value, const GsbRobustLossArgs *robust, float *loss_out3,
                             float *grad_rasterized_image, void *temp, int64_t temp_bytes, void *stream);
/* gsb200_train_step_filter3d with the weights: ... -> supervision pre-pass -> slice -> robust pre-passes on the image the
 * loss reads -> image loss on x' -> robust post-pass (dL/dx' -> dL/dx in place) -> slice backward -> supervision post-pass
 * -> ...  The depth, mask and feature terms are not weighted.  The pre- and post-passes run on a key-capacity overflow too;
 * they write only the weight, the composite and the stats, so the iteration stays a no-op.  NULL robust: exactly
 * gsb200_train_step_filter3d.  GSB_EINVAL, before any CUDA call, for robust not 0 or 1, a quantile outside (0, 1] or a
 * threshold outside [0, 1] with the robust mask, H or W not a multiple of 16, a NULL weight_out, composite or stats_out2,
 * a static weight, weight_out or composite not 4-byte aligned, a temp that is NULL, not 16-byte aligned or smaller
 * than gsb200_robust_temp_bytes, or a loss_temp of the train step that is not 16-byte aligned or smaller than
 * gsb200_image_loss_temp_bytes. */
int gsb200_train_step_robust(const GsbTrainStepArgs *args, const GsbSupervisionArgs *supervision,
                             const GsbFeatureTrainArgs *features, const GsbAppearanceArgs *appearance,
                             const GsbMcmcStepArgs *mcmc, const GsbFilter3dArgs *filter, const GsbRobustLossArgs *robust);
/* sizeof(GsbRobustLossArgs) */
void gsb200_abi_sizes_robust(int64_t *out1);

/* Individual stages (same workspace), for tests and profiling. */
int gsb200_stage_preprocess(const GsbForwardArgs *args);   /* K1+P1+K2+K3+P2+K4 fused */
int gsb200_stage_sort(const GsbForwardArgs *args);         /* P3 */
int gsb200_stage_tile_ranges(const GsbForwardArgs *args);  /* K5 */
int gsb200_stage_blend(const GsbForwardArgs *args);        /* K6 */

/* Diagnostic variants of forward/backward: identical launches with a CUDA event recorded on the
 * launching stream between stages; block until done and return device milliseconds per stage in
 * stage_ms_out[8] (host): forward = {empty (no workspace memset: the pose kernel clears the per-frame state), preprocess,
 * sort, tile ranges, blend};
 * backward = {grad/accumulator memsets, blend backward, per-point chain rule}.  (The reference's
 * counterpart is the Taichi kernel profiler, GaussianPointTrainer.py:217-219.) */
int gsb200_forward_timed(const GsbForwardArgs *args, float *stage_ms_out);
int gsb200_backward_timed(const GsbBackwardArgs *args, float *stage_ms_out);

/* Diagnostics: the blend kernels' real work, counted on the device (SURVEY 8(d) "E": pixel x splat evaluations).  Call after
 * gsb200_forward (same args / workspace; re-renders the same outputs) resp. after it with the backward args of the same frame
 * (adds into accum like gsb200_backward's loop A; pass a scratch accumulator).  host_out2[0] = (warp, splat) visits -- 32
 * pixel x splat evaluations each --, host_out2[1] = evaluations that contribute (alpha >= 1/255 on a live pixel).  The forward
 * variant fills 8 slots: [2..4] are what-if counters taken at staging time -- (patch, splat) pairs with the kernel's 8x4 patches,
 * with 8x8 patches (two pixels per thread) and with 16x4 patches -- the evidence for the patch shape in DESIGN.md.  Blocks.
 * (The reference's counterpart is the Taichi kernel profiler, GaussianPointTrainer.py:217-219.) */
int gsb200_forward_blend_work(const GsbForwardArgs *args, uint64_t *host_out8);
int gsb200_backward_blend_work(const GsbBackwardArgs *args, uint64_t *host_out2);

/* Checks the two hardware facts the default arithmetic path relies on: rcp.approx(1.0f) == 1.0f (a non-contributing
 * (pixel, splat) pair leaves the transmittance untouched in the branch-free backward, csrc/blend_bwd_transposed.cu) and
 * ex2.approx(0) == 1.  Returns GSB_OK or GSB_EUNSUPPORTED.  Blocks. */
int gsb200_device_selftest(void *stream);

/* find_tile_start_and_end, GPCR:175-193, on the reference's own key packing: sorted int64 keys
 * (tile << 32 | depth) -> [start, end) per tile; outputs must be zero-initialised (GPCR:954-957). */
int gsb200_find_tile_start_and_end(const int64_t *sorted_keys, int64_t num_keys, int32_t *tile_points_start,
                                   int32_t *tile_points_end, int32_t num_tiles, void *stream);

/* Stand-alone stable LSD radix sort of (key, int32 payload) pairs on the device; key_bytes 4 or 8,
 * bits [0, end_bit) are sorted.  temp must hold gsb200_sort_temp_bytes(n, key_bytes). Result is
 * left in keys_out / vals_out.  (Replaces torch.sort + gather, GPCR:947-950.) */
int64_t gsb200_sort_temp_bytes(int64_t n, int32_t key_bytes);
int gsb200_sort_pairs(const void *keys_in, const int32_t *vals_in, void *keys_out, int32_t *vals_out,
                      int64_t n, int32_t key_bytes, int32_t end_bit, void *temp, int64_t temp_bytes,
                      void *stream);

/* Host-buffer entry point (end-to-end inference call): the scene stays resident on the device, the
 * per-view inputs (pose, intrinsics) come from HOST memory and the image is returned to HOST memory.
 * host pointers should be pinned.  Blocks until the image is in host memory.
 * Replaces the render loop body gaussian_point_render.py:106-121 (pose .cuda(), forward, image .cpu()). */
int gsb200_render_host(const GsbForwardArgs *device_args, const float *host_q_pointcloud_camera,
                       const float *host_t_pointcloud_camera, const float *host_camera_intrinsics,
                       float *staging_device_pose /* >= num_objects*7+9 floats, device */,
                       float *host_image_out /* (H,W,3) */, int64_t *host_counters_out /* int64[4] or NULL */);

/* Fused clamp + L1 loss + gradient for the trainer step around the operator (SURVEY 8(f)-2):
 * loss = mean |clamp01(pred) - gt| (GaussianPointTrainer.py:168-170 clamp, LossFunction.py:29 L1) and, when
 * grad_predicted_out is not NULL, d(upstream_grad * loss)/d pred = upstream_grad * sign(.)/n inside the clamp
 * range, 0 outside -- what torch autograd produces with ~8 elementwise kernels.  All pointers are device
 * memory, 16-byte aligned; temp holds gsb200_l1_loss_temp_bytes() bytes and must be ZERO before its first use
 * (the call leaves it ready for the next one).  Deterministic (fixed grid, fixed summation order). */
int64_t gsb200_l1_loss_temp_bytes(void);
int gsb200_l1_loss(const float *predicted_image, const float *ground_truth_image, int64_t num_elements,
                   int32_t clamp01, float upstream_grad, float *loss_out, float *grad_predicted_out, void *temp,
                   int64_t temp_bytes, void *stream);

/* The trainer's whole image loss and its gradient (SURVEY 8(f)-2/3) in two kernels:
 *   pred = clamp(rasterized_image, 0, 1)                                  GaussianPointTrainer.py:168-170
 *   L    = (1 - lambda) * mean|pred - gt| + lambda * (1 - SSIM(pred, gt))  LossFunction.py:20-38
 * SSIM = the published pytorch_msssim algorithm the reference calls (LossFunction.py:4,31): 11-tap Gaussian window,
 * sigma 1.5, VALID padding, K = (0.01, 0.03), data_range 1, mean over the map.  rasterized_image is (H,W,3) as the
 * rasteriser returns it, ground_truth_image (3,H,W) as the dataset yields it; H, W > 10.  loss_out3 = {L, L1, 1 - SSIM};
 * grad_rasterized_image (H,W,3), if not NULL, receives upstream_grad * dL/d rasterized_image (zero where the clamp is
 * active).  temp holds gsb200_image_loss_temp_bytes(H, W) bytes, 16-byte aligned; its first 16 bytes must be ZERO before
 * the first use (the call leaves them ready for the next one).  Deterministic (fixed grid, fixed summation order).
 * Replaces ~60 autograd kernels per step (5 grouped convolutions, their transposes, ~25 elementwise). */
int64_t gsb200_image_loss_temp_bytes(int32_t camera_height, int32_t camera_width);
int gsb200_image_loss(const float *rasterized_image, const float *ground_truth_image, int32_t camera_height,
                      int32_t camera_width, float lambda_value, float upstream_grad, float *loss_out3,
                      float *grad_rasterized_image, void *temp, int64_t temp_bytes, void *stream);

/* One Adam step on a flat float32 tensor in ONE kernel (SURVEY 8(f)-2): the update of torch.optim.Adam as the reference
 * trainer configures it (GaussianPointTrainer.py:126-129: betas given, eps 1e-8, no weight decay, no amsgrad; stepped at
 * :176-177) -- m += (g - m)(1 - b1); v = v b2 + (1 - b2) g^2; p -= lr / (1 - b1^t) * m / (sqrt(v) / sqrt(1 - b2^t) + eps).
 * `step` is the 1-based step count t.  All pointers device memory, 16-byte aligned; exp_avg / exp_avg_sq are the
 * caller-owned state (zero before the first step).  lr / betas / eps are doubles like torch's Python floats (1 - beta is
 * formed in double).  HBM-bound: 28 B per element. */
int gsb200_adam_step(float *param, const float *grad, float *exp_avg, float *exp_avg_sq, int64_t num_elements, double lr,
                     double beta1, double beta2, double eps, int32_t step, void *stream);

/* The densification controller's per-iteration accumulator update in ONE kernel (SURVEY 8(f)-1): what
 * GaussianPointAdaptiveController.update does with the backward-hook tensors, GaussianPointAdaptiveController.py:130-143
 * (six indexed accumulations, mag / n_pixels with NaN -> 0, row norm; ~15 torch launches).  The first five arguments are
 * fields of BackwardValidPointHookInput (M entries), the last six the controller's accumulators (N entries; int32 / float32).
 * ids must be unique (they are: GPCR:861-864).  All pointers device memory. */
int gsb200_controller_update(const int32_t *point_id_in_camera_list, int64_t num_points_in_camera,
                             const int32_t *num_affected_pixels, const float *magnitude_grad_viewspace,
                             const float *grad_point_in_camera, int32_t *accumulated_num_in_camera,
                             int32_t *accumulated_num_pixels, float *accumulated_view_space_position_gradients,
                             float *accumulated_view_space_position_gradients_avg, float *accumulated_position_gradients,
                             float *accumulated_position_gradients_norm, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* GSB200_H_ */
