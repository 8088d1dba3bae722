// emu_mcmc.cpp -- the MCMC densification kernels (csrc/mcmc.cu) compiled as host C++ under simt_emu.h, launched as
// gsb200_mcmc_regulariser / gsb200_mcmc_noise / gsb200_mcmc_relocate launch them.  A library of its own.
// TEST INFRASTRUCTURE, see simt_emu.h.
#include "simt_emu.h"
#include "../../taichi_3d_gaussian_splatting_b200/csrc/mcmc.cu"

extern "C" long long emu_mcmc_temp_bytes() { return gsb::mcmc_temp_bytes(); }

// Returns the emulator's warp switches (> 0: the kernel ran its collectives).
extern "C" long long emu_mcmc_regulariser(const float *features, const signed char *invalid_mask, float *grad_features,
                                          long long N, long long num_valid, float lambda_opacity, float lambda_scale,
                                          float *terms_out2, void *temp) {
    using namespace gsb;
    simt_emu::M().switches = 0;
    const McmcRegulariserParams p = mcmc_regulariser_params(features, invalid_mask, grad_features, N, num_valid, lambda_opacity,
                                                            lambda_scale, terms_out2, temp);
    simt_emu::launch(mcmc_regulariser_kernel, mcmc_regulariser_blocks(N), MC_THREADS, p);
    return simt_emu::M().switches;
}

// skip: the value of the device flag the fused train step passes (non-zero = the launch is a no-op); < 0 = no flag
extern "C" void emu_mcmc_noise(float *pointcloud, const float *features, const signed char *invalid_mask, long long N,
                               float noise_scale, float gate_k, float min_opacity, unsigned long long seed, long long step,
                               long long skip) {
    using namespace gsb;
    McmcNoiseParams p = mcmc_noise_params(pointcloud, features, invalid_mask, N, noise_scale, gate_k, min_opacity, seed, step);
    p.skip_flag = skip >= 0 ? &skip : nullptr;
    simt_emu::launch(mcmc_noise_kernel, (int)((N + MC_THREADS - 1) / MC_THREADS), MC_THREADS, p);
}

extern "C" void emu_mcmc_relocate(const GsbMcmcRelocateArgs *a) {
    using namespace gsb;
    const McmcRelocateParams p = mcmc_relocate_params(*a);
    if (p.num_sources > 0)
        simt_emu::launch(mcmc_relocate_sources_kernel, (int)((p.num_sources + MC_THREADS - 1) / MC_THREADS), MC_THREADS, p);
    if (p.num_destinations > 0)
        simt_emu::launch(mcmc_relocate_copy_kernel, (int)((p.num_destinations + MC_WARPS - 1) / MC_WARPS), MC_THREADS, p);
}
