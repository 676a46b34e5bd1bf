// The prefiltered environment of the shading step's filtered mode (include/r3dg_b200.h, "PREFILTERED ENVIRONMENT"):
// the level table of a lat-long mip pyramid, shared by the pyramid build and adjoint (envfilter.cu) and the shading
// kernels (shading.cu), which read all levels as one texel array.
#pragma once
#include <cuda_runtime.h>

namespace r3dg {

#define ENV_MAX_LEVELS 16

struct EnvLevels {
    int L;                        // levels (1: the env has no coarser level and the mode changes nothing)
    int total;                    // texels over all levels
    float dtdp;                   // level 0: dtheta * dphi = (pi / (He - 1)) (2 pi / (We - 1))
    float sin_half;               // level 0: sin(dtheta / 2), the clamp of sin(theta) near the poles
    int h[ENV_MAX_LEVELS], w[ENV_MAX_LEVELS], off[ENV_MAX_LEVELS];   // rows, columns, first texel of each level
};

// Level l + 1 halves level l (ceil) in rows and columns while level l has at least 3 rows and 3 columns (so every level
// keeps at least 2 of each), up to ENV_MAX_LEVELS levels.
inline EnvLevels env_levels(int He, int We) {
    EnvLevels lv{};
    lv.L = 1; lv.h[0] = He; lv.w[0] = We; lv.off[0] = 0;
    while (lv.L < ENV_MAX_LEVELS && lv.h[lv.L - 1] >= 3 && lv.w[lv.L - 1] >= 3) {
        const int l = lv.L++;
        lv.h[l] = (lv.h[l - 1] + 1) / 2; lv.w[l] = (lv.w[l - 1] + 1) / 2;
        lv.off[l] = lv.off[l - 1] + lv.h[l - 1] * lv.w[l - 1];
    }
    lv.total = lv.off[lv.L - 1] + lv.h[lv.L - 1] * lv.w[lv.L - 1];
    if (lv.L > 1) {
        const double dt = 3.14159265358979323846 / (He - 1), dp = 2.0 * 3.14159265358979323846 / (We - 1);
        lv.dtdp = (float)(dt * dp);
        lv.sin_half = (float)sin(dt / 2.0);
    }
    return lv;
}

// envfilter.cu: dL/denv [He,We,3] = the adjoint of the pyramid applied to the gradient of all levels `g_pyr` (which it
// overwrites), in gather form without atomics: 2 launches per level above 0, or one copy for a one-level table
int launch_env_pyramid_adjoint(const EnvLevels& lv, float* g_pyr, float* d_env, cudaStream_t stream);

}  // namespace r3dg
