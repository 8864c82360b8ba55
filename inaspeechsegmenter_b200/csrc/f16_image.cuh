// f16_image.cuh -- host-only: fp32 weights [N][Kp] -> the tiled fp16 hi/lo operand image of engine 3 (conv_gemm_tc.cu).
// Kept free of CUDA runtime calls so that tools/f16_image_check.cu can exercise it on a machine without a GPU.
#pragma once
#include <cuda_fp16.h>
#include <math.h>

#include <vector>

// Layout: [n-tile][k-block of 64][hi | lo][BN rows x 128 bytes]; within a row the 16-byte chunk (8 halves)
// j is stored at chunk j ^ (row & 7) (SWIZZLE_128B, K-major -- the same convention as the TF32 image).
// Returns the power-of-two scale applied to the weights (max |w| * scale in [2^12, 2^13)).
static inline float iss_f16_build_image(const float *w, int N, int K, int Kp, int BN, std::vector<__half> &img)
{
    constexpr int HBK = 64;
    float maxabs = 0.f;
    for (int n = 0; n < N; ++n)
        for (int k = 0; k < K; ++k) maxabs = fmaxf(maxabs, fabsf(w[(size_t)n * Kp + k]));
    int e = 0;
    if (maxabs > 0.f) frexpf(maxabs, &e);                       // maxabs in [2^(e-1), 2^e)
    const float scale = ldexpf(1.f, 13 - e);
    const int nkb = K / HBK;
    img.assign((size_t)2 * N * K, __float2half_rn(0.f));
    for (int nt = 0; nt < N / BN; ++nt)
        for (int kb = 0; kb < nkb; ++kb) {
            const size_t base = (((size_t)nt * nkb + kb) * 2) * (size_t)BN * HBK;
            for (int n = 0; n < BN; ++n)
                for (int k = 0; k < HBK; ++k) {
                    const float v = w[(size_t)(nt * BN + n) * Kp + kb * HBK + k] * scale;
                    const __half h = __float2half_rn(v);
                    const __half l = __float2half_rn(v - __half2float(h));
                    const int chunk = (k >> 3) ^ (n & 7);
                    img[base + (size_t)n * HBK + chunk * 8 + (k & 7)] = h;
                    img[base + (size_t)BN * HBK + (size_t)n * HBK + chunk * 8 + (k & 7)] = l;
                }
        }
    return scale;
}
