// emu_robust.cpp -- the per-pixel loss weights of the fused train step (csrc/robust_loss.cu: histogram and mask pre-passes,
// then the image loss of csrc/image_loss.cu on the composite, then the post-pass) compiled as host C++ under simt_emu.h,
// chained as gsb200_robust_image_loss chains them.  A library of its own.  TEST INFRASTRUCTURE, see simt_emu.h.
#include "simt_emu.h"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/image_loss.cu"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/robust_loss.cu"

extern "C" long long emu_robust_temp_bytes() { return gsb::RL_TEMP_BYTES; }
extern "C" long long emu_robust_image_loss_temp_bytes(int H, int W) { return gsb::image_loss_layout(H, W).total; }

// image (H,W,3), gt (3,H,W), static_weight (H,W) or null; H, W multiples of 16.  Writes weight (H,W), composite (H,W,3),
// image_loss3 = {L, L1, 1 - SSIM} of (x', gt), grad_image = dL/dx (H,W,3) and stats2 = {inlier fraction, threshold}.
// Returns the emulator's warp switches (> 0: the kernels ran).
extern "C" long long emu_robust_step(const float *image, const float *gt, const float *static_weight, int H, int W,
                                     float lambda_value, int robust, float q, float box_threshold, float patch_threshold,
                                     float *weight, float *composite, float *image_loss3, float *grad_image, float *stats2,
                                     void *temp, void *image_loss_temp) {
    using namespace gsb;
    simt_emu::M().switches = 0;
    RobustParams rp;
    robust_params(image, gt, static_weight, H, W, robust, q, box_threshold, patch_threshold, weight, composite, grad_image,
                  temp, stats2, &rp);
    if (rp.robust) simt_emu::launch(robust_hist_kernel, robust_hist_blocks(H, W), RL_THREADS, rp);
    rp.counts[0] = rp.counts[1] = 0ull;  // launch_robust_pre's memset
    simt_emu::launch(robust_mask_kernel, (H / RL_TILE) * (W / RL_TILE), RL_THREADS, rp);
    ImageLossParams p;
    ImageLossLayout L;
    image_loss_params(composite, gt, H, W, lambda_value, 1.0f, image_loss3, grad_image, image_loss_temp, &p, &L);
    p.tiles_x = L.tiles_mx;
    p.tiles_y = L.tiles_my;
    simt_emu::launch(ssim_map_kernel, 3 * L.tiles_mx * L.tiles_my, IL_THREADS, p);
    p.tiles_x = L.tiles_ix;
    p.tiles_y = L.tiles_iy;
    simt_emu::launch(image_loss_grad_kernel, 3 * L.tiles_ix * L.tiles_iy, IL_THREADS, p);
    simt_emu::launch(robust_post_kernel, robust_post_blocks(H, W), RL_THREADS, rp);
    return simt_emu::M().switches;
}
