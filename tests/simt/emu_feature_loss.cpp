// emu_feature_loss.cpp -- the feature term of the fused train step (csrc/feature_loss.cu: the sum pass, then the gradient
// pass) compiled as host C++ under simt_emu.h, chained as gsb200_train_step_ext chains them.  A library of its own.
// TEST INFRASTRUCTURE, see simt_emu.h.
#include "simt_emu.h"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/feature_loss.cu"

extern "C" long long emu_feature_loss_temp_bytes() { return gsb::feature_loss_layout().total; }

template <int CP>
static void run(const gsb::FeatureLossParams &p, int blocks) {
    simt_emu::launch(gsb::feature_loss_sum_kernel<CP>, blocks, gsb::FL_THREADS, p);
    simt_emu::launch(gsb::feature_loss_grad_kernel<CP>, blocks, gsb::FL_THREADS, p);
}

// fmap (H,W,C); labels (H,W) for cross entropy, else target (H,W,C) for l2.  Writes grad (H,W,C) and
// loss2 = {feature term, n_supervised}.  Returns the emulator's warp switches (> 0: the kernels ran).
extern "C" long long emu_feature_loss(const float *fmap, const int *labels, const float *target, int H, int W, int C,
                                      float weight, float *grad, float *loss2, void *temp) {
    using namespace gsb;
    simt_emu::M().switches = 0;
    FeatureLossParams p;
    feature_loss_params(fmap, labels, target, H, W, C, weight, grad, loss2, temp, &p);
    const int blocks = feature_loss_blocks(H, W);
    switch (feature_loss_width(C)) {
        case 4: run<4>(p, blocks); break;
        case 8: run<8>(p, blocks); break;
        default: run<16>(p, blocks); break;
    }
    return simt_emu::M().switches;
}
