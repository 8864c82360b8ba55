// f16_image_check.cu -- host-only check of iss_f16_build_image (runs without a GPU):
//   * an independent reader that follows the wgmma shared-memory descriptor semantics (K-major, SWIZZLE_128B:
//     row r of a tile at byte r*128, 16-byte chunk c of that row at chunk c ^ (r & 7)) recovers B[n][k];
//   * (hi + lo) / scale reproduces every weight to 2^-21 relative or 2^-36 of the layer maximum (the fp16 subnormal floor after scaling);
//   * the scaled maximum lies in [2^12, 2^13).
//   nvcc -O2 -I../inaspeechsegmenter_b200/csrc -o /tmp/f16_image_check f16_image_check.cu && /tmp/f16_image_check
#include <cstdio>
#include <cstdlib>
#include <random>

#include "f16_image.cuh"

static float read_b(const std::vector<__half> &img, int N, int K, int BN, int n, int k, int part)
{
    const int nt = n / BN, r = n % BN, kb = k / 64, kk = k % 64, nkb = K / 64;
    const size_t stage = ((size_t)nt * nkb + kb) * 2 * (size_t)BN * 128;      // bytes: [hi tile | lo tile], BN rows x 128 B each
    const size_t tile = stage + (size_t)part * BN * 128;
    const int chunk = kk / 8, within = kk % 8;                                 // 8 halves per 16-byte chunk
    const size_t byte = tile + (size_t)r * 128 + (size_t)((chunk ^ (r & 7)) * 16) + within * 2;
    return __half2float(img[byte / 2]);
}

int main()
{
    std::mt19937 rng(7);
    int bad = 0;
    const int shapes[][3] = {{64, 1280, 64}, {128, 576, 128}, {128, 1152, 128}, {64, 128, 64}};
    for (auto &sh : shapes) {
        const int N = sh[0], K = sh[1], BN = sh[2], Kp = K;
        std::vector<float> w((size_t)N * Kp);
        std::normal_distribution<float> g(0.f, 0.03f);
        for (auto &v : w) v = g(rng);
        w[5] = 0.f; w[6] = 1e-9f; w[7] = -0.41f;
        std::vector<__half> img;
        const float scale = iss_f16_build_image(w.data(), N, K, Kp, BN, img);
        float maxabs = 0.f;
        for (float v : w) maxabs = fmaxf(maxabs, fabsf(v));
        if (!(maxabs * scale >= 4096.f && maxabs * scale < 8192.f)) { printf("scale out of range: %g\n", maxabs * scale); ++bad; }
        double worst_rel = 0, worst_abs = 0;
        for (int n = 0; n < N; ++n)
            for (int k = 0; k < K; ++k) {
                const double rec = ((double)read_b(img, N, K, BN, n, k, 0) + (double)read_b(img, N, K, BN, n, k, 1)) / scale;
                const double ref = w[(size_t)n * Kp + k];
                const double err = fabs(rec - ref);
                if (err > fabs(ref) * ldexp(1.0, -21) && err > maxabs * ldexp(1.0, -36)) ++bad;
                if (ref != 0) worst_rel = fmax(worst_rel, err / fabs(ref));
                worst_abs = fmax(worst_abs, err / maxabs);
            }
        printf("N=%d K=%d BN=%d: scale 2^%d, worst rel err %.2e, worst err / max|w| %.2e\n", N, K, BN, (int)log2f(scale), worst_rel, worst_abs);
    }
    printf(bad ? "FAILED (%d)\n" : "OK\n", bad);
    return bad != 0;
}
