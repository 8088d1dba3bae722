// emu_supervision_loss.cpp -- the supervision terms of the fused train step (csrc/supervision_loss.cu: pre-pass, then the
// image loss of csrc/image_loss.cu on the composited images, then the post-pass) compiled as host C++ under simt_emu.h,
// chained as gsb200_train_step_aux chains them.  A library of its own.  TEST INFRASTRUCTURE, see simt_emu.h.
#include "simt_emu.h"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/image_loss.cu"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/supervision_loss.cu"

extern "C" long long emu_supervision_temp_bytes(int H, int W) { return gsb::supervision_layout(H, W).total; }
extern "C" long long emu_supervision_image_loss_temp_bytes(int H, int W) { return gsb::image_loss_layout(H, W).total; }

// image (H,W,3), gt (3,H,W), alpha / depth (H,W); depth_target / mask_target / background may be null.  Writes
// image_loss3 = {L, L1, 1 - SSIM} of (I', gt'), grad_image = dL/dI (H,W,3), grad_alpha / grad_depth (H,W) where the terms
// are on, loss3 = {total, mask term, depth term}.  Returns the emulator's warp switches (> 0: the kernels ran).
extern "C" long long emu_supervision_step(const float *image, const float *gt, const float *alpha, const float *depth,
                                          const float *depth_target, const float *mask_target, const float *background,
                                          int H, int W, float lambda_value, float depth_weight, float mask_weight,
                                          float *image_loss3, float *grad_image, float *grad_alpha, float *grad_depth,
                                          float *loss3, void *temp, void *image_loss_temp) {
    using namespace gsb;
    simt_emu::M().switches = 0;
    SupervisionParams sp;
    supervision_params(image, gt, alpha, depth, depth_target, mask_target, background, H, W, depth_weight, mask_weight,
                       grad_image, grad_alpha, grad_depth, image_loss3, loss3, temp, &sp);
    const int blocks = supervision_blocks(H, W);
    simt_emu::launch(supervision_pre_kernel, blocks, SL_THREADS, sp);
    ImageLossParams p;
    ImageLossLayout L;
    image_loss_params(sp.image_out ? sp.image_out : image, sp.gt_out ? sp.gt_out : gt, H, W, lambda_value, 1.0f,
                      image_loss3, grad_image, image_loss_temp, &p, &L);
    p.tiles_x = L.tiles_mx;
    p.tiles_y = L.tiles_my;
    simt_emu::launch(ssim_map_kernel, 3 * L.tiles_mx * L.tiles_my, IL_THREADS, p);
    p.tiles_x = L.tiles_ix;
    p.tiles_y = L.tiles_iy;
    simt_emu::launch(image_loss_grad_kernel, 3 * L.tiles_ix * L.tiles_iy, IL_THREADS, p);
    simt_emu::launch(supervision_post_kernel, blocks, SL_THREADS, sp);
    return simt_emu::M().switches;
}
