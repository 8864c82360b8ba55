// conv_gemm.cuh -- implicit-GEMM convolution / dense layer shared by the CNN (K2)
// and ResNet101 (K5) operators.  NHWC float32 activations; B = [K][N] weights.
#pragma once
#include <cuda_fp16.h>

#include "iss_common.cuh"

// split-half word of the fp16-split engine: lo16 << 16 | hi16 with hi = fp16(x), lo = fp16(x - hi)
__device__ __forceinline__ uint32_t iss_pack_split(float y)
{
    const __half hh = __float2half_rn(y);
    const __half ll = __float2half_rn(y - __half2float(hh));
    return (uint32_t)__half_as_ushort(hh) | ((uint32_t)__half_as_ushort(ll) << 16);
}
// two values at once: the pair conversions map to F2FP (full-rate ALU) instead of the scalar F2F (conversion unit)
__device__ __forceinline__ void iss_pack_split2(float y0, float y1, uint32_t &w0, uint32_t &w1)
{
    const __half2 hh = __floats2half2_rn(y0, y1);
    const float2 hf = __half22float2(hh);
    const __half2 ll = __floats2half2_rn(y0 - hf.x, y1 - hf.y);
    const uint32_t h = *reinterpret_cast<const uint32_t *>(&hh), l = *reinterpret_cast<const uint32_t *>(&ll);
    w0 = __byte_perm(h, l, 0x5410);
    w1 = __byte_perm(h, l, 0x7632);
}
__device__ __forceinline__ float iss_unpack_split(uint32_t w)
{
    return __half2float(__ushort_as_half((unsigned short)(w & 0xFFFFu))) + __half2float(__ushort_as_half((unsigned short)(w >> 16)));
}

// ReLU with TensorFlow's NaN semantics: relu(NaN) = NaN.  fmaxf(NaN, 0) is 0, which would turn a non-finite activation
// (e.g. an fp16-split word past the fp16 range, hi = inf, lo = -inf) into a finite, wrong value downstream.
// max.NaN.f32 (sm_80+) is the same single instruction as fmaxf with NaN propagation; equal bits for every other input.
__device__ __forceinline__ float iss_relu(float v)
{
    float r;
    asm("max.NaN.f32 %0, %1, 0f00000000;" : "=f"(r) : "f"(v));
    return r;
}

#define ISS_F_RESIDUAL 64     /* internal: + residual[m][n] after the pre-affine, before ReLU */

// First layer folded into the operand fill of the convolution behind it (conv_gemm_tc.cu, LD_FIRST): the
// first Conv2D of the segmenter CNNs has ONE input channel and its input is the z-normalised patch
// (x - mu_j) / sigma_j (segmenter.py:82), so by linearity
//     conv(x^)[t, f, c] = (Y[row0_j + t, f, c] - mu_j * S_c) / sigma_j,   Y = conv(raw log-mel), S_c = sum of the filter
// and Y is shared by all the patches that overlap a frame (97 % overlap: hop 2 of 68 frames).  Y is computed once per
// batch in float64 and stored as a two-float number Yh + Yl (first_linear_kernel); bias and the BatchNorm affine
// (scale s_c, shift t_c) fold with the normalisation into ONE multiply-add per value,
//     a[t, f, c] = Y * alpha_jc + beta_jc,   alpha_jc = s_c / sigma_j,   beta_jc = (b_c s_c + t_c) - mu_j S_c alpha_jc,
// with alpha rounded to float32 FIRST and beta (float64, stored as two floats) computed from the rounded alpha, so the
// cancellation between Y alpha and beta is exact to ~1e-7 relative (first_coef_kernel).  The operand fill evaluates
// fma(Yh, alpha, beta_h) + fma(Yl, alpha, beta_l), ReLU, the optional second affine, and writes fp16 hi / lo planes
// straight into shared memory: the first layer's output (283 KB per patch, 47 % of all activation traffic) never
// exists in HBM.
struct FirstFuse {
    const float *Yh, *Yl;           // [y_rows][W * C] each, row r = conv of log-mel frames y_f0 + r ..; Y = Yh + Yl
    int64_t y_f0;                   // log-mel frame of Y row 0
    int64_t y_rows;
    const int32_t *row0;            // per patch of the batch: first log-mel frame
    const float *coef;              // per patch [3][C]: alpha, beta_hi, beta_lo
    const float *post_scale, *post_shift;   // first layer's affine behind the ReLU (nullptr = absent)
    int flags;                      // ISS_F_* of the first layer
    int64_t n_img;                  // patches in the batch
};

// A layer's weights as the tensor-core engines' operand images (conv_gemm_tc.cu), owned by the layer.  An image that
// is nullptr keeps the layer off that engine.
struct TcWeights {
    void *tiled = nullptr;          // engine 2: 3xTF32 hi / lo, tiled and swizzled as the shared-memory operand stages
    void *f16 = nullptr;            // engine 3: fp16 hi / lo, likewise, pre-scaled by a power of two
    float f16_inv_scale = 1.f;      // undoes that scale in the epilogue
};

struct ConvArgs {
    const float *in;        // NHWC activations, or the log-mel rows of the generic first layer
    const float *w;         // [K][N]
    const float *bias, *pre_scale, *pre_shift, *post_scale, *post_shift;
    const float *residual;  // [M][N] or nullptr
    float *out;             // [M][N]
    int64_t M;              // n_img * OH * OW
    int N, K;
    int H, W, C;            // input dims
    int OH, OW;
    int KH, KW, SH, SW, PT, PL;
    int flags;
    // generic first layer of the segmenter CNNs only (row0 != nullptr): gather the sliding patches from the log-mel
    // rows `in` (row stride ld) and z-normalise them on the fly
    int ld;
    const int32_t *row0; const float *mu; const float *sigma;
    TcWeights wt;
    // activation formats of engine 3: fp32 values (0) or split-half words lo16 << 16 | hi16 (1)
    int in_packed, out_packed;
    int residual_packed;    // `residual` holds split-half words (fp16-split kernels only)
    int pool_h, pool_w;     // engine 3 only, > 0: `in` is the un-pooled [n][pool_h][pool_w][C] tensor, 2x2 / stride-2 max taken in the operand fill
    const FirstFuse *first;         // host pointer, non-null: the fused first layer (copied into the kernel parameters)
};

// Epilogue coefficients of output channel n: bias, pre-affine (s1, t1), post-affine (s2, t2); absent terms are identities.
struct EpiCoef1 {
    float eb = 0.f, es1 = 1.f, et1 = 0.f, es2 = 1.f, et2 = 0.f;
};

__device__ __forceinline__ EpiCoef1 epi_coef1(const ConvArgs &a, int n)
{
    const bool pre = a.flags & ISS_F_AFFINE_PRE, post = a.flags & ISS_F_AFFINE_POST;
    EpiCoef1 c;
    c.eb = (a.flags & ISS_F_BIAS) ? __ldg(a.bias + n) : 0.f;
    c.es1 = pre ? __ldg(a.pre_scale + n) : 1.f;  c.et1 = pre ? __ldg(a.pre_shift + n) : 0.f;
    c.es2 = post ? __ldg(a.post_scale + n) : 1.f; c.et2 = post ? __ldg(a.post_shift + n) : 0.f;
    return c;
}

// The epilogue of the fp32 kernels: bias -> pre-affine -> (+ residual r) -> ReLU -> sigmoid -> post-affine.  Kernels that
// never take a residual (RESID = false) leave its test out, which keeps their register count.
template <bool RESID = false>
__device__ __forceinline__ float epi_f32(const EpiCoef1 &c, int flags, float acc, float r = 0.f)
{
    float v = acc + c.eb;
    if (flags & ISS_F_AFFINE_PRE) v = fmaf(v, c.es1, c.et1);
    if (RESID && (flags & ISS_F_RESIDUAL)) v += r;
    if (flags & ISS_F_RELU) v = iss_relu(v);
    if (flags & ISS_F_SIGMOID) v = 1.f / (1.f + expf(-v));
    if (flags & ISS_F_AFFINE_POST) v = fmaf(v, c.es2, c.et2);
    return v;
}

#define ISS_GEMM_FP32  0      /* fp32 CUDA cores (conv_gemm.cu) */
#define ISS_GEMM_TC_TS 2      /* wgmma 3xTF32 (conv_gemm_tc.cu): every layer shape with C, K, N multiples of 32 */
#define ISS_GEMM_TC_F16 3     /* wgmma fp16 hi/lo split (conv_gemm_tc.cu) for layers with C, N multiples of 64; other layers as engine 2 */
#ifndef ISS_GEMM_DEFAULT
#define ISS_GEMM_DEFAULT ISS_GEMM_TC_F16
#endif

extern "C" int iss_get_gemm_mode(void);

// Builds the tensor-core images of the weights W[K][N] (Keras / blob layout) of a layer with C input channels: engine 2's
// when C, K and N are multiples of 32, and engine 3's when `f16` is set and C and N are also multiples of 64.  These are
// the only shape rules of the two engines.  On failure the images already built stay in *w for iss_free_weights.
int iss_prepare_weights(const float *h_w, int C, int K, int N, bool f16, TcWeights *w);
void iss_free_weights(TcWeights *w);

// The kernel that runs a layer.  Only the engine-3 kernels (iss_conv_is_f16) read split-half words, take a folded
// pooling (pool_h > 0) or the fused first layer (`first`); they and the direct first-layer kernel write them
// (iss_conv_writes_words).  Layers with a sigmoid run on the fp32 kernels, the only ones that evaluate it.
enum IssConvKernel {
    ISS_CONV_F32,           // fp32 CUDA cores (conv_gemm.cu)
    ISS_CONV_F32_FIRST,     // the same, gathering the generic first layer's patches from the log-mel rows
    ISS_CONV_FIRST_DIRECT,  // first layer with one input channel and 16, 32, 64 or 128 outputs, one patch per CTA
    ISS_CONV_SMALL_N,       // fp32 dense / 1x1 layer with at most 8 outputs (the softmax heads)
    ISS_CONV_TF32,          // engine 2, gather kernel
    ISS_CONV_F16,           // engine 3, gather kernel
    ISS_CONV_F16_SLAB,      // engine 3, slab kernel
};
inline bool iss_conv_is_f16(IssConvKernel k) { return k == ISS_CONV_F16 || k == ISS_CONV_F16_SLAB; }
inline bool iss_conv_writes_words(IssConvKernel k) { return iss_conv_is_f16(k) || k == ISS_CONV_FIRST_DIRECT; }
IssConvKernel iss_conv_kernel(const ConvArgs &a, int mode);

// the tensor-core launchers behind iss_launch_conv (conv_gemm_tc.cu)
bool iss_slab_covers(const ConvArgs &a);
// rows of the gather kernel's shared-memory halo for a layer with the pooling folded in (0: global-memory fill)
int iss_gather_halo_rows(const ConvArgs &a);
// the same rows when the layer takes the pipelined path with two halos (0: it keeps another path)
int iss_gather_pipe_rows(const ConvArgs &a);
int iss_launch_conv_tf32(const ConvArgs &a, cudaStream_t st);
int iss_launch_conv_f16(const ConvArgs &a, cudaStream_t st);
int iss_launch_conv_slab(const ConvArgs &a, cudaStream_t st);

// Launches the layer on `st` with the kernel iss_conv_kernel(a, mode) picks.
int iss_launch_conv(const ConvArgs &a, int mode, cudaStream_t st);
