// emu_appearance.cpp -- the bilateral-grid kernels of csrc/appearance.cu (slice forward, slice backward with its finishing
// kernel, TV) compiled as host C++ under simt_emu.h and chained as launch_bilateral_grid_forward / _backward chain them.
// A library of its own.  TEST INFRASTRUCTURE, see simt_emu.h.
#include "simt_emu.h"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/appearance.cu"

extern "C" long long emu_bilateral_grid_temp_bytes(int H, int W, int gx, int gy, int gz) {
    return gsb::bilateral_grid_temp_bytes(H, W, gx, gy, gz);
}

// image (H,W,3), grid (12,Gz,Gy,Gx) -> out (H,W,3).  Returns the emulator's warp switches.
extern "C" long long emu_bilateral_grid_forward(const float *image, const float *grid, int H, int W, int gx, int gy, int gz,
                                                float *out) {
    using namespace gsb;
    simt_emu::M().switches = 0;
    BilateralGridParams p = {};
    bilateral_grid_shape(H, W, gx, gy, gz, &p);
    p.image = image;
    p.grid = grid;
    p.out = out;
    simt_emu::launch(bilateral_grid_forward_kernel, bilateral_grid_blocks(p), BG_THREADS, p);
    return simt_emu::M().switches;
}

// dL/dout (H,W,3) -> grad_in (H,W,3; may alias grad_out), grad_grid (12,Gz,Gy,Gx); with tv_out also the TV term
// (tv_weight) added into grad_grid and w tv in tv_out[0].  temp: emu_bilateral_grid_temp_bytes bytes.
extern "C" long long emu_bilateral_grid_backward(const float *image, const float *grid, int H, int W, int gx, int gy, int gz,
                                                 const float *grad_out, float *grad_in, float *grad_grid, void *temp,
                                                 float tv_weight, float *tv_out) {
    using namespace gsb;
    simt_emu::M().switches = 0;
    BilateralGridParams p = {};
    bilateral_grid_shape(H, W, gx, gy, gz, &p);
    p.image = image;
    p.grid = grid;
    p.grad_out = grad_out;
    p.grad_in = grad_in;
    p.partials = static_cast<float *>(temp);
    p.grad_grid = grad_grid;
    p.tv_out = tv_out;
    p.tv_weight = tv_weight;
    simt_emu::launch(bilateral_grid_backward_kernel, bilateral_grid_blocks(p), BG_THREADS, p);
    simt_emu::launch(bilateral_grid_finish_kernel, 3, BG_THREADS, p);  // any grid: the kernel strides over the node values
    if (tv_out) simt_emu::launch(bilateral_grid_tv_kernel, 1, TV_THREADS, p);
    return simt_emu::M().switches;
}
