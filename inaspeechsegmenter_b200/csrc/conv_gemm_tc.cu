// conv_gemm_tc.cu -- implicit-GEMM convolution / dense layer on the Hopper tensor cores (wgmma.mma_async, fp32
// accumulators in registers) with fp32-class accuracy, for every layer shape the tensor-core engines take: padded /
// strided / 1x1 convolutions (ResNet101), the KHxKW convolutions of the segmenter CNNs and Dense layers.
//
// Every fp32 operand x is split exactly into a high part and a low part and the product is accumulated as
//      A.B ~= Ah.Bh + Ah.Bl + Al.Bh          (dropped Al.Bl ~ 2^-22 relative)
// in two accumulators (D_main = Ah.Bh, D_lo = the two correction products) that are added in the epilogue.  Two engines:
//   engine 2 (3xTF32): hi = x with the 13 low mantissa bits cleared (a valid TF32 number), lo = x - hi; wgmma kind tf32.
//   engine 3 (fp16 split, the default): hi = fp16(x), lo = fp16(x - hi) (22 significant bits, like the TF32 split) on the
//       f16 tensor-core path, which runs at twice the TF32 rate.  The weights of a layer are pre-scaled by an exact power of
//       two so that max|w| lands in [2^12, 2^13) (undone in the epilogue); activations are used as they are, so
//       |activation| must stay below 65504 (true after BatchNorm / z-normalisation; a network that violates it must use
//       engine 2).
// Why the split: the reference evaluates its CNNs in fp32 and the parity bar is 1e-4 on the per-frame softmax; a single
// TF32 or fp16 pass (10-bit mantissa) misses it.
//
// PACKED activations ("split-half words", conv_gemm.cuh): a layer whose consumer is another engine-3 convolution stores
// every activation as ONE 32-bit word lo16 << 16 | hi16, so that the split is done once per element in the producing
// epilogue instead of KH*KW times in the consumers' operand fill.  The value carried between layers is hi + lo, exactly
// what the tensor cores would have used anyway.  Engine 3 also takes a 2x2 / stride-2 max-pooling in front of the
// convolution (the window maximum is taken in the operand fill, the pooling layer never runs) and the fused first layer of
// the segmenter CNNs (FirstFuse, conv_gemm.cuh: the first layer's output is evaluated in the operand fill from the
// float64 map Y and never exists in HBM).
//
// Tile: 128 output positions x BN output channels, K in blocks of one 128-byte operand row (32 TF32 / 64 fp16 values).
// Two warpgroups of 128 threads, each owns 64 GEMM rows: it gathers its rows of the k-block (im2col, one 16-byte chunk of
// the operand row per thread and row), splits them and writes hi / lo into a double-buffered SWIZZLE_128B tile, then
// issues its wgmmas.  The weights are static, so the host stores them already tiled and swizzled exactly as the shared
// memory operand image ([n-tile][k-block][hi|lo][BN rows x 128 B]); all 256 threads copy a stage with cp.async, four
// stages deep (two k-blocks ahead).  The global loads of k-block kb+1 are in flight while the wgmmas of kb are issued,
// and wgmma.wait_group 1 keeps one k-block of tensor work running while the next tile is filled.  The pooled instance
// (LD_POOL) launches 384 threads: where two tile halos fit it runs the persistent, warp-specialized gather_pipe, whose
// A operands come from the halo through ldmatrix into registers; elsewhere its warpgroups 1 and 2 run the loop above.
//
// The un-padded, stride-1 64 -> 64 convolutions of engine 3 (the segmenter CNNs' dominant 5x4 layer, with or without the
// fused first layer) run in conv_slab_kernel instead: it fills each input value once per tile into a "slab" whose
// row-shifted windows are the A operands of all taps, where the gather kernel above fills it once per tap.
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "conv_gemm.cuh"
#include "f16_image.cuh"
#include "tc_common.cuh"

namespace {

constexpr int TBM = 128, TBK = 32, HBK = 64;
constexpr int THREADS = 256;
constexpr int A_WG = 16384;                  // one warpgroup's operand tile of one stage: hi | lo, 64 rows x 128 B each
constexpr int A_STAGES = 2, B_STAGES = 4;
constexpr int MAX_SMEM = 227 * 1024;
// Tile halo of the pooled fill (LD_POOL) of 64 channels and more than one tap: every pooled input pixel the tile's output
// rows read, one word per channel.  The weight ring shrinks to three stages, one k-block ahead, to make room for it.
constexpr int HALO_PIX = 64 * 4;
constexpr int HALO_B_STAGES = 3;

constexpr int ENG_TF32 = 0, ENG_F16 = 1;
// operand fill of engine 3: fp32 values split here, split-half words, words with the 2x2 max-pooling in front (gather
// kernel only), or the fused first layer (slab kernel only).  Engine 2 reads fp32 values only.
constexpr int LD_F32 = 0, LD_PACKED = 1, LD_POOL = 2, LD_FIRST = 3;

template <int BN>
struct WgCfg {
    static constexpr int B_STAGE = 2 * BN * 128;                         // hi | lo, BN rows x 128 B each
    static constexpr int SMEM = B_STAGES * B_STAGE + A_STAGES * 2 * A_WG + 1024;
};

// shared memory of the gather kernel with a halo of `rows` input rows of width W
int halo_smem(int BN, int rows, int W)
{
    return HALO_B_STAGES * 2 * BN * 128 + A_STAGES * 2 * A_WG + 1024 + rows * W * HALO_PIX;
}

// Every launch of the pooled instance (LD_POOL) has 384 threads: on the pipelined path (gather_pipe) warpgroup 0 produces
// and warpgroups 1 and 2 consume; on the other paths warpgroup 0 gives its registers away and exits, and warpgroups 1 and
// 2 run the fill / wgmma loop of the other instances.
constexpr int POOL_THREADS = 384;
// the launch gives every thread 168 registers (384 threads, one CTA per SM): 128 x 24 + 256 x 240 = 128 x 112 + 256 x
// 192 = 384 x 168, so that setmaxnreg.inc finds the registers that setmaxnreg.dec released
constexpr int POOL_IDLE_REGS = 24, POOL_WG_REGS = 240;
constexpr int PIPE_PRODUCER_REGS = 112, PIPE_CONSUMER_REGS = 192;
constexpr int PIPE_FILL_THREADS = 96;                   // producer warps 1..3
constexpr int PIPE_CONSUMER_ARRIVALS = 8;               // lane 0 of each consumer warp
constexpr int PIPE_B_STAGES = 3, PIPE_HALOS = 2;
constexpr int PIPE_BAR_BYTES = 8 * 2 * (PIPE_B_STAGES + PIPE_HALOS);

// one halo buffer of the pipelined path: a hi plane and a lo plane of 128 bytes per pixel, for `rows` x W pixels and
// one zero pixel (the operand rows of padding and of rows past M point at it)
int pipe_halo_bytes(int rows, int W) { return 2 * (rows * W + 1) * 128; }
// its shared memory: the weight ring, two halo buffers, and 1024 bytes of alignment slack that also hold the mbarriers
int pipe_smem(int BN, int rows, int W) { return PIPE_B_STAGES * 2 * BN * 128 + PIPE_HALOS * pipe_halo_bytes(rows, W) + 1024; }

// The rows of a 128-row tile's halo: the rows g_lo .. g_lo + n - 1 of the batch as one tall pooled image (row img * H +
// ih), from the first input row of the tile's first output row to the last input row of its last one.
__device__ __forceinline__ void halo_span(const ConvArgs &a, int64_t tile, int64_t &g_lo, int &n)
{
    const int64_t ohw = (int64_t)a.OH * a.OW;
    const int64_t mf = tile * TBM, ml = (mf + TBM < a.M ? mf + TBM : a.M) - 1;
    const int64_t img0 = mf / ohw, img1 = ml / ohw;
    const int oh0 = (int)(mf - img0 * ohw) / a.OW, oh1 = (int)(ml - img1 * ohw) / a.OW;
    g_lo = img0 * a.H + max(oh0 * a.SH - a.PT, 0);
    n = (int)(img1 * a.H + min(oh1 * a.SH - a.PT + a.KH - 1, a.H - 1) - g_lo + 1);
}

// the four 2x2-window words of NW channels at the window offsets `offs` (words of `in`)
template <int NW>
__device__ __forceinline__ void pool_load(const uint32_t *in, const int64_t (&offs)[4], uint4 (&raw)[4][NW / 4])
{
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int h = 0; h < NW / 4; ++h) raw[q][h] = __ldg(reinterpret_cast<const uint4 *>(in + offs[q]) + h);
}

// 2x2 window maximum of split-half words: the WORD of the largest value is kept, as maxpool_nhwc_kernel<uint4> does:
// window order (0,0) (0,1) (1,0) (1,1), NaN wins, first maximum wins
template <int NW>
__device__ __forceinline__ void pool_select(const uint4 (&raw)[4][NW / 4], uint32_t (&bw)[NW])
{
    float bv[NW];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
#pragma unroll
        for (int h = 0; h < NW / 4; ++h) {
            const uint4 u = raw[q][h];
            const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float fv = iss_unpack_split(w[e]);
                if (q == 0 || fv > bv[4 * h + e] || fv != fv) { bv[4 * h + e] = fv; bw[4 * h + e] = w[e]; }
            }
        }
    }
}

// the same maximum of the words at the four window offsets `offs` (words of `in`), loaded and selected in one pass
template <int NW>
__device__ __forceinline__ void pool_max_words(const uint32_t *in, const int64_t (&offs)[4], uint32_t (&bw)[NW])
{
    float bv[NW];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
#pragma unroll
        for (int h = 0; h < NW / 4; ++h) {
            const uint4 u = __ldg(reinterpret_cast<const uint4 *>(in + offs[q]) + h);
            const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float fv = iss_unpack_split(w[e]);
                if (q == 0 || fv > bv[4 * h + e] || fv != fv) { bv[4 * h + e] = fv; bw[4 * h + e] = w[e]; }
            }
        }
    }
}

__device__ __forceinline__ void split_f16(const float (&v)[8], uint32_t (&hw)[4], uint32_t (&lw)[4])
{
#pragma unroll
    for (int e = 0; e < 4; ++e) {                            // hi = fp16(v), lo = fp16(v - hi): even k in the low half
        const __half2 hh = __floats2half2_rn(v[2 * e], v[2 * e + 1]);
        const float2 hf = __half22float2(hh);
        const __half2 ll = __floats2half2_rn(v[2 * e] - hf.x, v[2 * e + 1] - hf.y);
        hw[e] = *reinterpret_cast<const uint32_t *>(&hh);
        lw[e] = *reinterpret_cast<const uint32_t *>(&ll);
    }
}

__device__ __forceinline__ void words_to_planes(const uint32_t (&w)[8], uint32_t (&hw)[4], uint32_t (&lw)[4])
{
#pragma unroll
    for (int e = 0; e < 4; ++e) {                            // word = lo << 16 | hi; operand column = k even (low) | k odd (high)
        hw[e] = __byte_perm(w[2 * e], w[2 * e + 1], 0x5410);
        lw[e] = __byte_perm(w[2 * e], w[2 * e + 1], 0x7632);
    }
}

// Epilogue of both kernels for the output pair (m, nb), (m, nb + 1): inv_scale (engine 3), bias, pre-affine, residual,
// ReLU, post-affine, then fp32 values or split-half words.
struct EpiCoef {
    float eb[2], es1[2], et1[2], es2[2], et2[2];
};

__device__ __forceinline__ EpiCoef epi_coef(const ConvArgs &a, int nb)
{
    const bool has_bias = a.flags & ISS_F_BIAS, pre = a.flags & ISS_F_AFFINE_PRE, post = a.flags & ISS_F_AFFINE_POST;
    EpiCoef c;
#pragma unroll
    for (int q = 0; q < 2; ++q) {
        c.eb[q] = has_bias ? __ldg(a.bias + nb + q) : 0.f;
        c.es1[q] = pre ? __ldg(a.pre_scale + nb + q) : 1.f;  c.et1[q] = pre ? __ldg(a.pre_shift + nb + q) : 0.f;
        c.es2[q] = post ? __ldg(a.post_scale + nb + q) : 1.f; c.et2[q] = post ? __ldg(a.post_shift + nb + q) : 0.f;
    }
    return c;
}

template <int ENG>
__device__ __forceinline__ void epi_store(const ConvArgs &a, const EpiCoef &c, int64_t m, int nb, float y0, float y1, float inv_scale)
{
    const bool pre = a.flags & ISS_F_AFFINE_PRE, post = a.flags & ISS_F_AFFINE_POST;
    const bool relu = a.flags & ISS_F_RELU, resid = a.flags & ISS_F_RESIDUAL;
    float y[2] = {y0, y1};
    float rv[2] = {0.f, 0.f};
    if (resid) {
        const uint2 rw = __ldg(reinterpret_cast<const uint2 *>(a.residual + m * a.N + nb));
        if (a.residual_packed) { rv[0] = iss_unpack_split(rw.x); rv[1] = iss_unpack_split(rw.y); }
        else { rv[0] = __uint_as_float(rw.x); rv[1] = __uint_as_float(rw.y); }
    }
#pragma unroll
    for (int q = 0; q < 2; ++q) {
        float v;
        if constexpr (ENG == ENG_F16)                         // ((acc * inv_s) + bias) * s1 + t1 as one multiply-add
            v = fmaf(y[q], inv_scale * c.es1[q], fmaf(c.eb[q], c.es1[q], c.et1[q]));
        else {
            v = y[q] + c.eb[q];
            if (pre) v = fmaf(v, c.es1[q], c.et1[q]);
        }
        if (resid) v += rv[q];
        if (relu) v = iss_relu(v);
        if (post) v = fmaf(v, c.es2[q], c.et2[q]);
        y[q] = v;
    }
    float *dst = a.out + m * a.N + nb;
    if (a.out_packed) *reinterpret_cast<uint2 *>(dst) = make_uint2(iss_pack_split(y[0]), iss_pack_split(y[1]));
    else *reinterpret_cast<float2 *>(dst) = make_float2(y[0], y[1]);
}

// The same epilogue for the single engine-3 output (m, n) (the slab kernel, whose accumulator rows are channels), with
// the coefficients of epi_coef1 (conv_gemm.cuh).
__device__ __forceinline__ void epi_store1(const ConvArgs &a, const EpiCoef1 &c, int64_t m, int n, float y, float inv_scale)
{
    float v = fmaf(y, inv_scale * c.es1, fmaf(c.eb, c.es1, c.et1));
    if (a.flags & ISS_F_RESIDUAL) {
        const uint32_t rw = __ldg(reinterpret_cast<const uint32_t *>(a.residual + m * a.N + n));
        v += a.residual_packed ? iss_unpack_split(rw) : __uint_as_float(rw);
    }
    if (a.flags & ISS_F_RELU) v = iss_relu(v);
    if (a.flags & ISS_F_AFFINE_POST) v = fmaf(v, c.es2, c.et2);
    float *dst = a.out + m * a.N + n;
    if (a.out_packed) *reinterpret_cast<uint32_t *>(dst) = iss_pack_split(v);
    else *dst = v;
}

// epilogue of one warpgroup's 64 rows m0 .. m0 + 63 (thread t of the warpgroup) from its accumulators: hh + (hl + lh)
template <int ENG, int BN>
__device__ __forceinline__ void wg_epilogue(const ConvArgs &a, const float (&dm)[BN / 2], const float (&dl)[BN / 2], int64_t m0,
                                            int n0, int t, float inv_scale)
{
    const int w = t >> 5, l = t & 31;
    const int64_t mr = m0 + 16 * w + (l >> 2);
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
        const int nb = n0 + 8 * i + 2 * (l & 3);
        const EpiCoef c = epi_coef(a, nb);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int64_t m = mr + 8 * h;
            if (m >= a.M) continue;
            epi_store<ENG>(a, c, m, nb, dm[4 * i + 2 * h] + dl[4 * i + 2 * h], dm[4 * i + 2 * h + 1] + dl[4 * i + 2 * h + 1], inv_scale);
        }
    }
}

// ============================ pipelined pooled path (LD_POOL, C = 64, two halos fit) ============================
// Persistent: CTA i takes the 128-row tiles i, i + gridDim.x, ... in increasing order (so CTAs running at the same time
// share input rows in L2).  Warpgroup 0 produces: its warp 0 streams the weight stage of every k-block (one tap of 64
// channels) with one bulk copy into a three-stage ring, its warps 1..3 stage the halo of the next tile into the other of
// two halo buffers.  A halo buffer holds the pooled pixel p of the tile's rows (halo_span) as a hi plane and a lo plane
// of 128 bytes each, 16-byte chunk q (channels 8 q .. 8 q + 7) at chunk q ^ (p & 7), so that 8 consecutive pixels hit all
// 32 banks.  Warpgroups 1 and 2 consume 64 output rows each: per k16 step each warp gathers its 16 im2col rows from the
// halo with one ldmatrix.x4 for hi and one for lo (lane l gives row (l & 7) + 8 ((l >> 3) & 1), chunk 2 kk + l / 16)
// and issues Ah.Bh, Ah.Bl and Al.Bh with A in registers: the same products in the same order as the other paths, into
// the same two accumulators.  Full / empty mbarriers hand every weight stage and every halo buffer over.
template <int BN>
__device__ __forceinline__ void gather_pipe(const ConvArgs &a, const unsigned char *__restrict__ wt, float inv_scale, int halo_rows)
{
    constexpr int B_STAGE = WgCfg<BN>::B_STAGE;
    extern __shared__ unsigned char smem_dyn[];
    const uint32_t base = smem_u32(smem_dyn);
    const uint32_t ring = (base + 1023u) & ~1023u;
    const uint32_t halo0 = ring + (uint32_t)PIPE_B_STAGES * B_STAGE;
    const int zp = halo_rows * a.W;                                     // the zero pixel
    const uint32_t plane = (uint32_t)(zp + 1) * 128u, halo_bytes = 2 * plane;
    const uint32_t bars = ring - base >= (uint32_t)PIPE_BAR_BYTES ? base : halo0 + PIPE_HALOS * halo_bytes;
    const uint32_t wfull = bars, wempty = bars + 8 * PIPE_B_STAGES;                       // + 8 * stage
    const uint32_t hfull = bars + 16 * PIPE_B_STAGES, hempty = hfull + 8 * PIPE_HALOS;     // + 8 * buffer

    const int tid = threadIdx.x, wg = tid >> 7;
    if (tid == 0) {
        for (int s = 0; s < PIPE_B_STAGES; ++s) { mbar_init(wfull + 8 * s, 1); mbar_init(wempty + 8 * s, PIPE_CONSUMER_ARRIVALS); }
        for (int b = 0; b < PIPE_HALOS; ++b) { mbar_init(hfull + 8 * b, PIPE_FILL_THREADS); mbar_init(hempty + 8 * b, PIPE_CONSUMER_ARRIVALS); }
        fence_mbar_init();
    }
    if (tid < 2 * PIPE_HALOS * 8) {                                     // the zero pixel of both planes of both buffers
        const int q = tid & 7, pl = tid >> 3;
        sts128(halo0 + (uint32_t)(pl >> 1) * halo_bytes + (uint32_t)(pl & 1) * plane + (uint32_t)zp * 128u + q * 16, 0u, 0u, 0u, 0u);
    }
    __syncthreads();

    const int nkb = a.KH * a.KW;                                        // one k-block (64 channels) per tap
    const int64_t tiles = (a.M + TBM - 1) / TBM;
    const unsigned char *wtile = wt + (size_t)blockIdx.y * nkb * B_STAGE;

    if (wg == 0) {
        // ============================ producer ============================
        setmaxnreg_dec<PIPE_PRODUCER_REGS>();
        if (tid < 32) {                                                 // warp 0: the weight stage of every k-block
            if (tid == 0) {
                int s = 0;
                uint32_t ph = 0;
                for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x)
                    for (int kb = 0; kb < nkb; ++kb) {
                        mbar_wait(wempty + 8 * s, ph ^ 1);              // both consumers retired the wgmmas that read it
                        mbar_arrive_expect_tx(wfull + 8 * s, B_STAGE);
                        bulk_copy_g2s(ring + (uint32_t)s * B_STAGE, wtile + (size_t)kb * B_STAGE, B_STAGE, wfull + 8 * s);
                        if (++s == PIPE_B_STAGES) { s = 0; ph ^= 1; }
                    }
            }
        } else {                                                        // warps 1..3: the halo of every tile
            const uint32_t *in = reinterpret_cast<const uint32_t *>(a.in);
            const int ft = tid - 32;
            int b = 0;
            uint32_t ph = 0;
            for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
                int64_t g_lo;
                int n;
                halo_span(a, tile, g_lo, n);
                mbar_wait(hempty + 8 * b, ph ^ 1);                      // both consumers read their last tap from it
                const uint32_t hi = halo0 + (uint32_t)b * halo_bytes, lo = hi + plane;
                // units (pixel, 16-byte chunk q of 8 channels), two per thread in flight
                const int nu = n * a.W * 8;
#pragma unroll 1
                for (int u0 = ft; u0 < nu; u0 += 2 * PIPE_FILL_THREADS) {
                    uint4 raw[2][4][2];
#pragma unroll
                    for (int v = 0; v < 2; ++v) {
                        const int u = u0 + v * PIPE_FILL_THREADS;
                        if (u < nu) {
                            const int64_t gp = g_lo * a.W + (u >> 3);   // pixel of the tall pooled image
                            const int64_t gr = gp / a.W, img = gr / a.H;
                            const int iw = (int)(gp - gr * a.W), ih = (int)(gr - img * a.H);
                            const int64_t p00 = ((img * a.pool_h + 2 * ih) * a.pool_w + 2 * iw) * a.C + (u & 7) * 8;
                            const int64_t offs[4] = {p00, p00 + a.C, p00 + (int64_t)a.pool_w * a.C, p00 + (int64_t)a.pool_w * a.C + a.C};
                            pool_load<8>(in, offs, raw[v]);
                        }
                    }
#pragma unroll
                    for (int v = 0; v < 2; ++v) {
                        const int u = u0 + v * PIPE_FILL_THREADS;
                        if (u < nu) {
                            uint32_t w[8], hw[4], lw[4];
                            pool_select<8>(raw[v], w);
                            words_to_planes(w, hw, lw);
                            const int px = u >> 3, q = u & 7;
                            const uint32_t o = (uint32_t)px * 128u + ((uint32_t)(q ^ (px & 7)) << 4);
                            sts128(hi + o, hw[0], hw[1], hw[2], hw[3]);
                            sts128(lo + o, lw[0], lw[1], lw[2], lw[3]);
                        }
                    }
                }
                mbar_arrive(hfull + 8 * b);
                if (++b == PIPE_HALOS) { b = 0; ph ^= 1; }
            }
        }
        return;
    }

    // ============================ consumers ============================
    setmaxnreg_inc<PIPE_CONSUMER_REGS>();
    const int c = wg - 1, t = tid & 127, w = t >> 5, l = t & 31;
    const int r = 16 * w + (l & 7) + 8 * ((l >> 3) & 1);               // this lane's ldmatrix row of the warpgroup's 64
    const int half = l >> 4;                                            // and its 16-byte half of each k16 step
    const int n0 = blockIdx.y * BN;
    int s = 0, b = 0;
    uint32_t wph = 0, hph = 0;
    for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        int64_t g_lo;
        int n;
        halo_span(a, tile, g_lo, n);
        const int64_t m0 = tile * TBM + 64 * c, m = m0 + r;
        const bool okr = m < a.M;
        const int64_t ohw = (int64_t)a.OH * a.OW;
        const int64_t img = okr ? m / ohw : 0;
        const int rem = okr ? (int)(m - img * ohw) : 0;
        const int oh = rem / a.OW, ow = rem - oh * a.OW;
        const int ih0 = oh * a.SH - a.PT, iw0 = ow * a.SW - a.PL, hb = (int)(img * a.H - g_lo);

        float dm[BN / 2], dl[BN / 2];
#pragma unroll
        for (int q = 0; q < BN / 2; ++q) { dm[q] = 0.f; dl[q] = 0.f; }
        wgmma_fence_operand(dm);
        wgmma_fence_operand(dl);
        mbar_wait(hfull + 8 * b, hph);
        const uint32_t hi = halo0 + (uint32_t)b * halo_bytes;

        int kh = 0, kw = 0;
        for (int kb = 0; kb < nkb; ++kb) {
            const int ih = ih0 + kh, iw = iw0 + kw;
            const int p = okr && ih >= 0 && ih < a.H && iw >= 0 && iw < a.W ? (hb + ih) * a.W + iw : zp;
            uint32_t ah[4][4], al[4][4];
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const uint32_t o = hi + (uint32_t)p * 128u + ((uint32_t)((2 * kk + half) ^ (p & 7)) << 4);
                ldsm_x4(o, ah[kk]);
                ldsm_x4(o + plane, al[kk]);
            }
            if (kb == nkb - 1) {                                        // the last read of this halo buffer
                __syncwarp();
                if (l == 0) mbar_arrive(hempty + 8 * b);
            }
            mbar_wait(wfull + 8 * s, wph);                              // the weights of this tap landed
            wgmma_fence();
            const uint64_t db = make_sw128_desc(ring + (uint32_t)s * B_STAGE), dbl = db + ((BN * 128) >> 4);
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                wgmma_f16_rs<BN>(dm, ah[kk], db + 2 * kk);              // Ah.Bh
                wgmma_f16_rs<BN>(dl, ah[kk], dbl + 2 * kk);             // Ah.Bl
                wgmma_f16_rs<BN>(dl, al[kk], db + 2 * kk);              // Al.Bh
            }
            wgmma_commit();
            wgmma_wait<0>();                                            // the A registers and the stage are free again
            if (l == 0) mbar_arrive(wempty + 8 * s);
            if (++s == PIPE_B_STAGES) { s = 0; wph ^= 1; }
            if (++kw == a.KW) { kw = 0; ++kh; }
        }
        wgmma_fence_operand(dm);
        wgmma_fence_operand(dl);
        if (++b == PIPE_HALOS) { b = 0; hph ^= 1; }
        wg_epilogue<ENG_F16, BN>(a, dm, dl, m0, n0, t, inv_scale);
    }
}

// halo_rows > 0 (LD_POOL with C = 64 only): the tile's pooled input rows fit in a halo of that many rows.  The tile then
// takes the 2x2 maximum of each of them once, stages the words in shared memory and fills every tap from there instead of
// taking the maximum of four global words per tap and value.  pipe (LD_POOL only): two such halos fit, and the layer runs
// on the pipelined path gather_pipe.
template <int ENG, int BN, int MODE>
__global__ void __launch_bounds__(MODE == LD_POOL ? POOL_THREADS : THREADS, 1)
conv_gemm_wg_kernel(const ConvArgs a, const unsigned char *__restrict__ wt, float inv_scale, int halo_rows, int pipe)
{
    using Cfg = WgCfg<BN>;
    constexpr int KE = ENG == ENG_F16 ? HBK : TBK;                       // k-elements per block
    constexpr int RAW = ENG == ENG_F16 ? 2 : 1;                          // 16-byte input loads per 16-byte operand chunk
    constexpr bool PREFETCH = MODE == LD_F32 || MODE == LD_PACKED;       // raw input held in registers one k-block ahead
    if constexpr (MODE == LD_POOL) {
        static_assert(ENG == ENG_F16, "the pooled fill is an engine-3 fill");
        if (pipe) { gather_pipe<BN>(a, wt, inv_scale, halo_rows); return; }
        if (threadIdx.x < 128) { setmaxnreg_dec<POOL_IDLE_REGS>(); return; }
        setmaxnreg_inc<POOL_WG_REGS>();
    }
    // the 256 threads of the fill / wgmma loop (warpgroups 1 and 2 of the pooled instance) and their barrier
    auto fill_sync = [&]() {
        if constexpr (MODE == LD_POOL) asm volatile("bar.sync 1, 256;" ::: "memory");
        else __syncthreads();
    };
    const bool halo = MODE == LD_POOL && halo_rows > 0;
    const int b_stages = halo ? HALO_B_STAGES : B_STAGES, b_ahead = b_stages - 2;
    extern __shared__ unsigned char smem_dyn[];
    unsigned char *smem = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    unsigned char *b_ring = smem;
    const uint32_t b_ring_u32 = smem_u32(b_ring);
    const uint32_t a_ring_u32 = b_ring_u32 + (uint32_t)b_stages * Cfg::B_STAGE;
    const uint32_t halo_u32 = a_ring_u32 + A_STAGES * 2 * A_WG;

    const int tid = threadIdx.x - (MODE == LD_POOL ? 128 : 0), wg = tid >> 7, t = tid & 127;
    const int64_t m0 = (int64_t)blockIdx.x * TBM + wg * 64;
    const int n0 = blockIdx.y * BN;
    const int nkb = a.K / KE;
    const unsigned char *wtile = wt + (size_t)blockIdx.y * nkb * Cfg::B_STAGE;

    auto issue_b = [&](int kb) {
        if (kb < nkb) {
            const unsigned char *src = wtile + (size_t)kb * Cfg::B_STAGE;
            const uint32_t dst = b_ring_u32 + (uint32_t)(kb % b_stages) * Cfg::B_STAGE;
#pragma unroll
            for (int o = tid * 16; o < Cfg::B_STAGE; o += THREADS * 16) cp_async16_u32(dst + o, src + o, 16);
        }
        cp_async_commit();                                   // (empty groups keep the group count uniform)
    };
    for (int kb = 0; kb < b_ahead; ++kb) issue_b(kb);

    // this thread's operand rows (64 per warpgroup): r_i = t / 8 + 16 i, 16-byte chunk j of the 128-byte operand row
    const int j = t & 7;
    int row_img[4], row_ih0[4], row_iw0[4];
    uint32_t ok_mask = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int64_t m = m0 + (t >> 3) + 16 * i;
        const bool okr = m < a.M;
        ok_mask |= (okr ? 1u : 0u) << i;
        const int64_t mm = okr ? m : 0;
        const int64_t ohw = (int64_t)a.OH * a.OW;
        const int64_t img = mm / ohw;
        const int rem = (int)(mm - img * ohw);
        const int oh = rem / a.OW, ow = rem - oh * a.OW;
        row_img[i] = (int)img;
        row_ih0[i] = oh * a.SH - a.PT;
        row_iw0[i] = ow * a.SW - a.PL;
    }
    const uint32_t row_dst0 = (uint32_t)((t >> 3) * 128 + ((j ^ ((t >> 3) & 7)) << 4));   // (t/8 + 16 i) & 7 == (t/8) & 7
    // The halo holds the pixels of the rows g_lo .. g_lo + halo_n - 1 of the batch as one tall image (row img * H + ih):
    // from the first input row of the tile's first output row to the last input row of its last one.  Row i's pixel
    // (ih, iw) is halo pixel (row_hb[i] + ih) * W + iw.
    int64_t g_lo = 0;
    int halo_n = 0, row_hb[4];
    if (halo) {
        halo_span(a, blockIdx.x, g_lo, halo_n);
#pragma unroll
        for (int i = 0; i < 4; ++i) row_hb[i] = (int)((int64_t)row_img[i] * a.H - g_lo);
    }
    if constexpr (MODE == LD_POOL) {
        if (halo) {                                          // stage the halo: 16 chunks of 16 bytes per pixel
            const int nu = halo_n * a.W * 16;
#pragma unroll 4
            for (int u = tid; u < nu; u += THREADS) {
                const int px = u >> 4, q = u & 15;
                const int64_t gp = g_lo * a.W + px;          // pixel of the tall pooled image
                const int64_t gr = gp / a.W, img = gr / a.H;
                const int iw = (int)(gp - gr * a.W), ih = (int)(gr - img * a.H);
                const int64_t p00 = ((img * a.pool_h + 2 * ih) * a.pool_w + 2 * iw) * a.C + q * 4;
                const int64_t offs[4] = {p00, p00 + a.C, p00 + (int64_t)a.pool_w * a.C, p00 + (int64_t)a.pool_w * a.C + a.C};
                uint32_t w[4];
                pool_max_words(reinterpret_cast<const uint32_t *>(a.in), offs, w);
                sts128(halo_u32 + (uint32_t)u * 16u, w[0], w[1], w[2], w[3]);
            }
            fill_sync();
        }
    }
    // tap of the next k-block to fill: k = (rr * KW + ss) * C + c0
    int tap_c0 = 0, tap_ss = 0, tap_rr = 0;
    auto advance = [&]() {
        tap_c0 += KE;
        if (tap_c0 == a.C) { tap_c0 = 0; if (++tap_ss == a.KW) { tap_ss = 0; ++tap_rr; } }
    };
    auto pixel_ok = [&](int i, int &ih, int &iw) {
        ih = row_ih0[i] + tap_rr; iw = row_iw0[i] + tap_ss;
        return ((ok_mask >> i) & 1u) && ih >= 0 && ih < a.H && iw >= 0 && iw < a.W;
    };

    uint4 raw[4][RAW];
    auto fetch = [&]() {                                     // PREFETCH modes: the raw 16-byte chunks of the next k-block
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            int ih, iw;
            if (pixel_ok(i, ih, iw)) {
                const uint4 *p = reinterpret_cast<const uint4 *>(
                    a.in + (((int64_t)row_img[i] * a.H + ih) * a.W + iw) * a.C + tap_c0 + j * (4 * RAW));
#pragma unroll
                for (int q = 0; q < RAW; ++q) raw[i][q] = __ldg(p + q);
            } else {
#pragma unroll
                for (int q = 0; q < RAW; ++q) raw[i][q] = make_uint4(0u, 0u, 0u, 0u);
            }
        }
        advance();
    };

    // split the k-block into the hi / lo tiles of stage s of this warpgroup
    auto fill = [&](int s) {
        const uint32_t hi_base = a_ring_u32 + (uint32_t)(s * 2 + wg) * A_WG, lo_base = hi_base + A_WG / 2;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t dst = row_dst0 + i * 16 * 128;
            uint32_t hw[4], lw[4];
            if constexpr (ENG == ENG_TF32) {
                const uint32_t v[4] = {raw[i][0].x, raw[i][0].y, raw[i][0].z, raw[i][0].w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    hw[e] = v[e] & 0xFFFFE000u;
                    lw[e] = __float_as_uint(__uint_as_float(v[e]) - __uint_as_float(hw[e]));
                }
            } else if constexpr (MODE == LD_F32) {
                const float v[8] = {__uint_as_float(raw[i][0].x), __uint_as_float(raw[i][0].y), __uint_as_float(raw[i][0].z), __uint_as_float(raw[i][0].w),
                                    __uint_as_float(raw[i][1].x), __uint_as_float(raw[i][1].y), __uint_as_float(raw[i][1].z), __uint_as_float(raw[i][1].w)};
                split_f16(v, hw, lw);
            } else if constexpr (MODE == LD_PACKED) {
                const uint32_t w[8] = {raw[i][0].x, raw[i][0].y, raw[i][0].z, raw[i][0].w, raw[i][1].x, raw[i][1].y, raw[i][1].z, raw[i][1].w};
                words_to_planes(w, hw, lw);
            } else {
                static_assert(MODE == LD_POOL, "the fused first layer runs in conv_slab_kernel");
                // the 2x2 window of the un-pooled NHWC tensor [img][pool_h][pool_w][C]: the WORD of the largest value is kept
                // (as maxpool_nhwc_kernel<uint4> does: window order (0,0) (0,1) (1,0) (1,1), NaN wins, first maximum wins)
                uint32_t bw[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
                int ih, iw;
                if (pixel_ok(i, ih, iw) && halo) {
                    // the 8 words of chunk j from the halo; threads j >= 4 read their two 16-byte halves in the other
                    // order, so that the 8 chunks of a quarter warp hit all 32 banks
                    const uint32_t p = halo_u32 + (uint32_t)((row_hb[i] + ih) * a.W + iw) * HALO_PIX + j * 32;
                    const uint32_t sw = (uint32_t)(j & 4) << 2;
                    const uint4 x = lds128(p + sw), y = lds128(p + (sw ^ 16u));
                    const uint4 u0 = sw ? y : x, u1 = sw ? x : y;
                    bw[0] = u0.x; bw[1] = u0.y; bw[2] = u0.z; bw[3] = u0.w; bw[4] = u1.x; bw[5] = u1.y; bw[6] = u1.z; bw[7] = u1.w;
                } else if (pixel_ok(i, ih, iw)) {
                    const int64_t p00 = (((int64_t)row_img[i] * a.pool_h + 2 * ih) * a.pool_w + 2 * iw) * a.C + tap_c0 + j * 8;
                    const int64_t offs[4] = {p00, p00 + a.C, p00 + (int64_t)a.pool_w * a.C, p00 + (int64_t)a.pool_w * a.C + a.C};
                    pool_max_words(reinterpret_cast<const uint32_t *>(a.in), offs, bw);
                }
                words_to_planes(bw, hw, lw);
            }
            sts128(hi_base + dst, hw[0], hw[1], hw[2], hw[3]);
            sts128(lo_base + dst, lw[0], lw[1], lw[2], lw[3]);
        }
        if constexpr (!PREFETCH) advance();
    };

    float dm[BN / 2], dl[BN / 2];
#pragma unroll
    for (int q = 0; q < BN / 2; ++q) { dm[q] = 0.f; dl[q] = 0.f; }

    if constexpr (PREFETCH) fetch();
    for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb & 1;
        fill(s);                                             // stage s was last read by this warpgroup's wgmmas of kb - 2
        if constexpr (PREFETCH) { if (kb + 1 < nkb) fetch(); }
        if (halo) cp_async_wait<0>();                        // weights of kb landed
        else cp_async_wait<1>();                             // (kb + 1 may still be in flight)
        fence_proxy_async();
        fill_sync();
        issue_b(kb + b_ahead);                              // its stage was read by kb - 2, retired in every warpgroup
        wgmma_fence();
        const uint64_t da = make_sw128_desc(a_ring_u32 + (uint32_t)(s * 2 + wg) * A_WG);
        const uint64_t dal = da + ((A_WG / 2) >> 4);
        const uint64_t db = make_sw128_desc(b_ring_u32 + (uint32_t)(kb % b_stages) * Cfg::B_STAGE);
        const uint64_t dbl = db + ((BN * 128) >> 4);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {                     // 32 bytes of the operand row per wgmma (k16 fp16 / k8 tf32)
            if constexpr (ENG == ENG_F16) {
                wgmma_f16<BN>(dm, da + 2 * kk, db + 2 * kk);     // Ah.Bh
                wgmma_f16<BN>(dl, da + 2 * kk, dbl + 2 * kk);    // Ah.Bl
                wgmma_f16<BN>(dl, dal + 2 * kk, db + 2 * kk);    // Al.Bh
            } else {
                wgmma_tf32<BN>(dm, da + 2 * kk, db + 2 * kk);
                wgmma_tf32<BN>(dl, da + 2 * kk, dbl + 2 * kk);
                wgmma_tf32<BN>(dl, dal + 2 * kk, db + 2 * kk);
            }
        }
        wgmma_commit();
        wgmma_wait<1>();
    }
    wgmma_wait<0>();
    cp_async_wait<0>();

    wg_epilogue<ENG, BN>(a, dm, dl, m0, n0, t, inv_scale);
}

template <int ENG, int BN, int MODE>
int launch_wg(const ConvArgs &a, const void *wt, float inv_scale, cudaStream_t st)
{
    using Cfg = WgCfg<BN>;
    auto kern = conv_gemm_wg_kernel<ENG, BN, MODE>;
    const int pipe_rows = MODE == LD_POOL ? iss_gather_pipe_rows(a) : 0;
    const int halo_rows = pipe_rows > 0 ? pipe_rows : MODE == LD_POOL ? iss_gather_halo_rows(a) : 0;
    const int smem = pipe_rows > 0 ? pipe_smem(BN, pipe_rows, a.W) : halo_rows > 0 ? halo_smem(BN, halo_rows, a.W) : Cfg::SMEM;
    ISS_CUDA_OK(iss_optin_smem(reinterpret_cast<const void *>(kern), smem));
    const int64_t gm = (a.M + TBM - 1) / TBM;
    ISS_REQUIRE(gm < (1ll << 31), ISS_ERR_INVALID, "conv_tc: M too large");
    dim3 grid((unsigned)gm, (unsigned)(a.N / BN));
    if (pipe_rows > 0) {                                     // persistent: at most one CTA per SM and n-tile
        int dev = 0, sms = 0;
        ISS_CUDA_OK(cudaGetDevice(&dev));
        ISS_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        grid.x = (unsigned)(gm < sms ? gm : sms);
    }
    const int threads = MODE == LD_POOL ? POOL_THREADS : THREADS;
    kern<<<grid, threads, smem, st>>>(a, reinterpret_cast<const unsigned char *>(wt), inv_scale, halo_rows, pipe_rows > 0);
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch();
    return ISS_OK;
}

// ============================ slab kernel: un-padded, stride-1 engine-3 convolutions with C = N = 64 ============================
// The input of a batch is read as ONE tall image, pixel p = (img * H + ih) * W + iw, and every output slot gets the same
// numbering, s = (img * H + oh) * W + ow.  The operand of tap (kh, kw) for the slots s0 .. s0 + 127 is then the 128
// consecutive pixels from s0 + kh * W + kw.  A tile is the slots s0 .. s0 + 255; its pixels
// s0 .. s0 + 255 + (KH - 1) W + KW - 1 are evaluated, split and stored once into a SWIZZLE_128B hi plane and lo plane
// (the "slab"), and every tap's slot operand is a row-shifted window of it, addressed by the wgmma descriptor alone.  So
// each input value is filled about 1.3 times instead of KH * KW times.  Slots with oh >= OH or ow >= OW (and slots past
// the batch) are computed and not stored.  Slab rows past the last pixel of the batch are zero.
// The slots are the N side of the products and the 64 output channels the M side: the weight stage of a tap is the
// engine-3 image [hi: 64 rows | lo: 64 rows] x 128 B, whose halves are the A operands Bh^T and Bl^T, and a consumer's 128
// slots are one N = 128 window.  So the three products hh = Bh^T.Ah, hl = Bl^T.Ah and lh = Bh^T.Al are three
// m64n128k16 per k16 step, each reading 6 KB of shared memory for 64 tensor clocks (with the slots on the M side they
// were an m64n128 Ah.[Bh | Bl] and an m64n64 Al.Bh per 64 slots, 10 KB for 96 clocks, and the n64 shape alone needs the
// whole 128 B/clk of shared-memory bandwidth).  Each accumulator element still sums the same products of one slot and
// one channel in the same order, and the epilogue adds hh + (hl + lh) as before.
//
// The kernel is persistent and warp-specialized: one CTA per SM takes tiles blockIdx.x, blockIdx.x + gridDim.x, ... (in
// increasing order, so neighbouring CTAs share the first-layer map and input rows in L2).  Warpgroup 0 produces: its
// warp 0 streams the weight stage of every tap with one bulk copy into a ring of `stages` stages, its warps 1..3 fill the
// slab of the next tile into one of `nbuf` slab buffers.  Warpgroups 1 and 2 consume: consumer c owns the slots
// s0 + 128 c .. s0 + 128 c + 127 and issues, per tap, the wgmmas above.  Full / empty mbarriers hand every weight stage
// and every slab buffer from producer to consumers and back.  setmaxnreg moves registers from the producer (which holds
// no accumulators) to the consumers (3 x 64 accumulator registers each).  With two slab buffers the fill of tile t + 1
// runs while the consumers compute tile t; where two slabs do not fit (tall filters) one buffer is refilled once both
// consumers have retired their last wgmma on it.
constexpr int SLAB_TS = 256, SLAB_C = 64, SLAB_N = 64;
constexpr int SLAB_THREADS = 384;                       // producer warpgroup + two consumer warpgroups
constexpr int SLAB_FILL_THREADS = 96;                   // producer warps 1..3
constexpr int SLAB_CONSUMER_ARRIVALS = 8;               // lane 0 of each consumer warp
// the launch gives every thread 168 registers (384 threads, one CTA per SM): 128 x 56 + 256 x 224 = 384 x 168
constexpr int SLAB_PRODUCER_REGS = 56, SLAB_CONSUMER_REGS = 224;
constexpr int SLAB_B_STAGE = 2 * SLAB_N * 128;          // hi | lo, 64 rows x 128 B each
constexpr int SLAB_MAX_STAGES = 4, SLAB_MAX_BUF = 2;
constexpr int SLAB_BAR_BYTES = 8 * 2 * (SLAB_MAX_STAGES + SLAB_MAX_BUF);
constexpr int SLAB_MAX_SMEM = MAX_SMEM;

// slab rows of a tile (a multiple of 8, so that the lo plane stays 1024-byte aligned) and the kernel's shared memory:
// `stages` weight stages, `nbuf` slabs and 1024 bytes of alignment slack, which also hold the mbarriers
int slab_rows(int KH, int KW, int W) { return (SLAB_TS + (KH - 1) * W + KW - 1 + 7) & ~7; }
int slab_smem(int rows, int nbuf, int stages) { return stages * SLAB_B_STAGE + nbuf * 2 * rows * 128 + 1024; }

// One 16-byte chunk of the slab, chunk j of pixel row r (pixel p = s0 + r = (img * H + ih) * W + iw): slab_load issues
// the global loads of the chunk's 8 channels (for LD_FIRST the map Y of the pixel's own patch; zeros past the batch),
// slab_store evaluates, splits and stores them at chunk j ^ (r & 7) of both planes.
struct SlabRaw {
    uint4 x[4];                                               // LD_FIRST: Yh (x[0..1]) and Yl (x[2..3]); else x[0..1]
};

template <int MODE>
__device__ __forceinline__ void slab_load(const ConvArgs &a, const FirstFuse &ff, int64_t p, int64_t img, int ih, int iw,
                                          int j, bool ok, SlabRaw &raw)
{
#pragma unroll
    for (int q = 0; q < 4; ++q) raw.x[q] = make_uint4(0u, 0u, 0u, 0u);
    if (!ok) return;
    if constexpr (MODE == LD_FIRST) {
        const int64_t o = (((int64_t)__ldg(ff.row0 + img) - ff.y_f0 + ih) * a.W + iw) * SLAB_C + j * 8;
        const uint4 *yh = reinterpret_cast<const uint4 *>(ff.Yh + o), *yl = reinterpret_cast<const uint4 *>(ff.Yl + o);
        raw.x[0] = __ldg(yh); raw.x[1] = __ldg(yh + 1); raw.x[2] = __ldg(yl); raw.x[3] = __ldg(yl + 1);
    } else {                                                  // NHWC pixel p of the batch is the tall image's pixel p
        const uint4 *src = reinterpret_cast<const uint4 *>(a.in + p * SLAB_C + j * 8);
        raw.x[0] = __ldg(src); raw.x[1] = __ldg(src + 1);
    }
}

template <int MODE>
__device__ __forceinline__ void slab_store(const FirstFuse &ff, const SlabRaw &raw, int64_t img, int j, bool ok, uint32_t slab_hi,
                                           uint32_t slab_lo, int r)
{
    uint32_t hw[4] = {0u, 0u, 0u, 0u}, lw[4] = {0u, 0u, 0u, 0u};
    if (ok) {
        if constexpr (MODE == LD_FIRST) {                     // the first layer at the pixel
            const float4 *cf = reinterpret_cast<const float4 *>(ff.coef + img * (3 * SLAB_C) + j * 8);
            float v[8];
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                const uint4 h4 = raw.x[q], l4 = raw.x[2 + q];
                const float4 va = __ldg(cf + q), vh = __ldg(cf + SLAB_C / 4 + q), vl = __ldg(cf + 2 * (SLAB_C / 4) + q);
                const float hv[4] = {__uint_as_float(h4.x), __uint_as_float(h4.y), __uint_as_float(h4.z), __uint_as_float(h4.w)};
                const float lv[4] = {__uint_as_float(l4.x), __uint_as_float(l4.y), __uint_as_float(l4.z), __uint_as_float(l4.w)};
                const float al[4] = {va.x, va.y, va.z, va.w}, bh[4] = {vh.x, vh.y, vh.z, vh.w}, bl[4] = {vl.x, vl.y, vl.z, vl.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    float x = fmaf(hv[e], al[e], bh[e]) + fmaf(lv[e], al[e], bl[e]);
                    if (ff.flags & ISS_F_RELU) x = iss_relu(x);
                    if (ff.flags & ISS_F_AFFINE_POST) {
                        const int c = j * 8 + 4 * q + e;
                        x = fmaf(x, __ldg(ff.post_scale + c), __ldg(ff.post_shift + c));
                    }
                    v[4 * q + e] = x;
                }
            }
            split_f16(v, hw, lw);
        } else {
            const uint4 u0 = raw.x[0], u1 = raw.x[1];
            if constexpr (MODE == LD_PACKED) {
                const uint32_t w[8] = {u0.x, u0.y, u0.z, u0.w, u1.x, u1.y, u1.z, u1.w};
                words_to_planes(w, hw, lw);
            } else {
                static_assert(MODE == LD_F32, "slab fill modes: LD_F32, LD_PACKED, LD_FIRST");
                const float v[8] = {__uint_as_float(u0.x), __uint_as_float(u0.y), __uint_as_float(u0.z), __uint_as_float(u0.w),
                                    __uint_as_float(u1.x), __uint_as_float(u1.y), __uint_as_float(u1.z), __uint_as_float(u1.w)};
                split_f16(v, hw, lw);
            }
        }
    }
    const uint32_t dst = (uint32_t)r * 128u + ((uint32_t)(j ^ (r & 7)) << 4);
    sts128(slab_hi + dst, hw[0], hw[1], hw[2], hw[3]);
    sts128(slab_lo + dst, lw[0], lw[1], lw[2], lw[3]);
}

// (img, ih, iw) of the pixel n rows of the tall image further on (n >= 0)
__device__ __forceinline__ void slab_step(const ConvArgs &a, int n, int64_t &img, int &ih, int &iw)
{
    iw += n;
    while (iw >= a.W) { iw -= a.W; if (++ih == a.H) { ih = 0; ++img; } }
}

// The slab of the tile at slot s0, filled by fill thread ft of 96: chunk j = ft % 8 of the pixel rows ft / 8 + 12 i.
// The thread walks its pixels' (img, ih, iw) from one division per tile instead of dividing the 64-bit pixel index
// for every row: the fill sets the pace of the layer, and those divisions were most of its dependent instructions.
// (Keeping two rows' loads in flight instead spills the LD_FIRST producer at 56 registers and was slower.)
template <int MODE>
__device__ __forceinline__ void slab_fill(const ConvArgs &a, const FirstFuse &ff, uint32_t slab_hi, uint32_t slab_lo, int rows,
                                          int64_t s0, int ft, int64_t HW, int64_t n_img)
{
    constexpr int STEP = SLAB_FILL_THREADS / 8;                // rows between a thread's rows
    const int j = ft & 7;
    int r = ft >> 3;
    int64_t img = (s0 + r) / HW;
    const int rem = (int)(s0 + r - img * HW);
    int ih = rem / a.W, iw = rem - ih * a.W;
#pragma unroll 1
    for (; r < rows; r += STEP) {
        const bool ok0 = img < n_img;
        SlabRaw raw0;
        slab_load<MODE>(a, ff, s0 + r, img, ih, iw, j, ok0, raw0);
        slab_store<MODE>(ff, raw0, img, j, ok0, slab_hi, slab_lo, r);
        slab_step(a, STEP, img, ih, iw);
    }
}

template <int MODE>
__global__ void __launch_bounds__(SLAB_THREADS, 1)
conv_slab_kernel(const ConvArgs a, const FirstFuse ff, const unsigned char *__restrict__ wt, float inv_scale, int rows,
                 int64_t tiles, int nbuf, int stages)
{
    extern __shared__ unsigned char smem_dyn[];
    const uint32_t base = smem_u32(smem_dyn);
    const uint32_t ring = (base + 1023u) & ~1023u;           // weight stages, then the slabs: 1024-byte aligned
    const uint32_t slab0 = ring + (uint32_t)stages * SLAB_B_STAGE, slab_bytes = (uint32_t)rows * 256u;
    // the mbarriers go into the bytes the alignment skips when they fit there, else right after the slabs: either way
    // inside the 1024 bytes of slack that slab_smem counts
    const uint32_t bars = ring - base >= (uint32_t)SLAB_BAR_BYTES ? base : slab0 + (uint32_t)nbuf * slab_bytes;
    const uint32_t wfull = bars, wempty = bars + 8 * SLAB_MAX_STAGES;                   // + 8 * stage
    const uint32_t sfull = bars + 16 * SLAB_MAX_STAGES, sempty = sfull + 8 * SLAB_MAX_BUF;  // + 8 * buffer

    const int tid = threadIdx.x, wg = tid >> 7;
    if (tid == 0) {
        for (int s = 0; s < stages; ++s) { mbar_init(wfull + 8 * s, 1); mbar_init(wempty + 8 * s, SLAB_CONSUMER_ARRIVALS); }
        for (int b = 0; b < nbuf; ++b) { mbar_init(sfull + 8 * b, SLAB_FILL_THREADS); mbar_init(sempty + 8 * b, SLAB_CONSUMER_ARRIVALS); }
        fence_mbar_init();
    }
    __syncthreads();

    const int nkb = a.KH * a.KW;                             // one k-block (64 channels) per tap
    const int64_t HW = (int64_t)a.H * a.W;
    const int64_t n_img = a.M / ((int64_t)a.OH * a.OW);

    if (wg == 0) {
        // ============================ producer ============================
        setmaxnreg_dec<SLAB_PRODUCER_REGS>();
        if (tid < 32) {                                      // warp 0: the weight stages of every tap of every tile
            if (tid == 0) {
                int s = 0;
                uint32_t ph = 0;
                for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x)
                    for (int kb = 0; kb < nkb; ++kb) {
                        mbar_wait(wempty + 8 * s, ph ^ 1);   // both consumers retired the wgmmas that read the stage
                        mbar_arrive_expect_tx(wfull + 8 * s, SLAB_B_STAGE);
                        bulk_copy_g2s(ring + (uint32_t)s * SLAB_B_STAGE, wt + (size_t)kb * SLAB_B_STAGE, SLAB_B_STAGE, wfull + 8 * s);
                        if (++s == stages) { s = 0; ph ^= 1; }
                    }
            }
        } else {                                             // warps 1..3: the slab of every tile
            int b = 0;
            uint32_t ph = 0;
            for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
                mbar_wait(sempty + 8 * b, ph ^ 1);           // both consumers retired their last wgmma on this buffer
                const uint32_t hi = slab0 + (uint32_t)b * slab_bytes, lo = hi + (uint32_t)rows * 128u;
                slab_fill<MODE>(a, ff, hi, lo, rows, tile * SLAB_TS, tid - 32, HW, n_img);
                fence_proxy_async();                         // this thread's slab stores, visible to wgmma
                mbar_arrive(sfull + 8 * b);
                if (++b == nbuf) { b = 0; ph ^= 1; }
            }
        }
        return;
    }

    // ============================ consumers ============================
    setmaxnreg_inc<SLAB_CONSUMER_REGS>();
    const int c = wg - 1, t = tid & 127, w = t >> 5, l = t & 31;
    int s = 0, b = 0;
    uint32_t wph = 0, sph = 0;
    for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int64_t s0 = tile * SLAB_TS;
        // the consumer's 128 slots as the N side of three m64n128 products, output channels as the M side:
        // hh = Bh^T.Ah, hl = Bl^T.Ah, lh = Bh^T.Al (accumulator row = channel, column = slot)
        float hh[SLAB_N], hl[SLAB_N], lh[SLAB_N];
#pragma unroll
        for (int q = 0; q < SLAB_N; ++q) { hh[q] = 0.f; hl[q] = 0.f; lh[q] = 0.f; }
        wgmma_fence_operand(hh);                             // keep the zeroing out of the wgmma pipeline (ptxas would
        wgmma_fence_operand(hl);                             // otherwise serialize every wgmma of the loop)
        wgmma_fence_operand(lh);
        mbar_wait(sfull + 8 * b, sph);
        const uint32_t slab_hi = slab0 + (uint32_t)b * slab_bytes, slab_lo = slab_hi + (uint32_t)rows * 128u;

        int kh = 0, kw = 0, prev = -1;
        for (int kb = 0; kb < nkb; ++kb) {
            mbar_wait(wfull + 8 * s, wph);                   // the weights of this tap landed
            wgmma_fence();
            const uint32_t stage = ring + (uint32_t)s * SLAB_B_STAGE;
            const uint64_t dwh = make_sw128_desc(stage), dwl = make_sw128_desc(stage + SLAB_N * 128);
            const int row = 128 * c + kh * a.W + kw;
            const uint64_t dxh = make_sw128_desc_rows(slab_hi, row), dxl = make_sw128_desc_rows(slab_lo, row);
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                wgmma_f16<2 * SLAB_N>(hh, dwh + 2 * kk, dxh + 2 * kk);
                wgmma_f16<2 * SLAB_N>(hl, dwl + 2 * kk, dxh + 2 * kk);
                wgmma_f16<2 * SLAB_N>(lh, dwh + 2 * kk, dxl + 2 * kk);
            }
            wgmma_commit();
            wgmma_wait<1>();                                 // the previous tap's wgmmas retired: release its stage
            if (prev >= 0 && l == 0) mbar_arrive(wempty + 8 * prev);
            prev = s;
            if (++s == stages) { s = 0; wph ^= 1; }
            if (++kw == a.KW) { kw = 0; ++kh; }
        }
        wgmma_wait<0>();
        wgmma_fence_operand(hh);
        wgmma_fence_operand(hl);
        wgmma_fence_operand(lh);
        if (l == 0) { mbar_arrive(wempty + 8 * prev); mbar_arrive(sempty + 8 * b); }
        if (++b == nbuf) { b = 0; sph ^= 1; }

        // ---- epilogue: register q = 4 i + 2 h + e holds channel 16 w + l / 4 + 8 h of slot
        //      s0 + 128 c + 8 i + 2 (l % 4) + e, stored only when the slot is an output position ----
        EpiCoef1 cf[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) cf[h] = epi_coef1(a, 16 * w + (l >> 2) + 8 * h);
        const int64_t sl0 = s0 + 128 * c + 2 * (l & 3);
        int64_t img = sl0 / HW;                              // (img, oh, ow) of slot sl0 + 8 i, advanced with i
        int rem = (int)(sl0 - img * HW);
        int oh = rem / a.W, ow = rem - oh * a.W;
#pragma unroll
        for (int i = 0; i < 2 * SLAB_N / 8; ++i) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                int64_t ie = img;
                int he = oh, we = ow + e;
                if (we == a.W) { we = 0; if (++he == a.H) { he = 0; ++ie; } }
                if (ie < n_img && he < a.OH && we < a.OW) {
                    const int64_t m = (ie * a.OH + he) * a.OW + we;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int q = 4 * i + 2 * h + e;
                        epi_store1(a, cf[h], m, 16 * w + (l >> 2) + 8 * h, hh[q] + (hl[q] + lh[q]), inv_scale);
                    }
                }
            }
            ow += 8;
            while (ow >= a.W) { ow -= a.W; if (++oh == a.H) { oh = 0; ++img; } }
        }
    }
}

template <int MODE>
int launch_slab(const ConvArgs &a, cudaStream_t st)
{
    const int rows = slab_rows(a.KH, a.KW, a.W);
    // two slabs (the fill of the next tile overlaps the current one) and a three-stage ring where they fit, else one
    // slab and four stages
    const bool pingpong = slab_smem(rows, 2, 3) <= SLAB_MAX_SMEM;
    const int nbuf = pingpong ? 2 : 1, stages = pingpong ? 3 : SLAB_MAX_STAGES, smem = slab_smem(rows, nbuf, stages);
    auto kern = conv_slab_kernel<MODE>;
    ISS_CUDA_OK(iss_optin_smem(reinterpret_cast<const void *>(kern), smem));
    const int64_t n_img = a.M / ((int64_t)a.OH * a.OW);
    const int64_t slots = ((n_img - 1) * a.H + a.OH - 1) * (int64_t)a.W + a.OW;    // through the last output position
    const int64_t tiles = (slots + SLAB_TS - 1) / SLAB_TS;
    int dev = 0, sms = 0;
    ISS_CUDA_OK(cudaGetDevice(&dev));
    ISS_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const unsigned grid = (unsigned)(tiles < sms ? tiles : sms);
    const FirstFuse ff = a.first ? *a.first : FirstFuse{};
    kern<<<grid, SLAB_THREADS, smem, st>>>(a, ff, reinterpret_cast<const unsigned char *>(a.wt.f16), a.wt.f16_inv_scale, rows,
                                           tiles, nbuf, stages);
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch();
    return ISS_OK;
}

template <int BN>
int launch_f16(const ConvArgs &a, cudaStream_t st)
{
    const float s = a.wt.f16_inv_scale;
    if (a.pool_h > 0) return launch_wg<ENG_F16, BN, LD_POOL>(a, a.wt.f16, s, st);
    if (a.in_packed) return launch_wg<ENG_F16, BN, LD_PACKED>(a, a.wt.f16, s, st);
    return launch_wg<ENG_F16, BN, LD_F32>(a, a.wt.f16, s, st);
}

// n-tile width of engine 3: 128 output channels per CTA when N allows it, else 64 (the weight image and the launch agree)
int f16_bn_for(int N) { return N % 128 == 0 ? 128 : 64; }

// n-tile width of engine 2
int tf32_bn_for(int N) { return N % 128 == 0 ? 128 : (N % 64 == 0 ? 64 : 32); }

int upload(const void *h, size_t bytes, void **d_out, const char *what)
{
    void *d = nullptr;
    cudaError_t e = cudaMalloc(&d, bytes);
    if (e != cudaSuccess) { iss_set_error("cudaMalloc %s: %s", what, cudaGetErrorString(e)); return ISS_ERR_NOMEM; }
    e = cudaMemcpy(d, h, bytes, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) { cudaFree(d); iss_set_error("cudaMemcpy %s: %s", what, cudaGetErrorString(e)); return ISS_ERR_CUDA; }
    *d_out = d;
    return ISS_OK;
}

int g_gemm_mode = -1;      // -1 = read ISS_B200_GEMM on first use

}  // namespace

// Input rows (of the batch as one tall image, row img * H + ih) that the 128 output rows of one tile read, at most over
// every tile start: tiles start at multiples of 128, i.e. at the positions s * gcd(128, OH * OW) of an image.
extern "C" int iss_gather_halo_rows_bound(int H, int OH, int OW, int KH, int SH, int PT)
{
    const int64_t ohw = (int64_t)OH * OW;
    int64_t g = TBM, r = ohw;
    while (r) { const int64_t q = g % r; g = r; r = q; }
    int64_t rows = 0;
    for (int64_t s = 0; s < ohw; s += g) {
        const int64_t last = s + TBM - 1, img1 = last / ohw;
        const int64_t oh0 = s / OW, oh1 = (last - img1 * ohw) / OW;
        const int64_t lo = std::max<int64_t>(oh0 * SH - PT, 0), hi = img1 * H + std::min<int64_t>(oh1 * SH - PT + KH - 1, H - 1);
        rows = std::max(rows, hi - lo + 1);
    }
    return (int)rows;
}

// Shared memory of a gather-kernel layer with the pooling folded in (LD_POOL) when it takes the halo, 0 for the
// global-memory fill: the halo holds one 64-channel block (C = 64), filters with one tap reuse no input, and the halo
// must fit in shared memory next to the rings.
extern "C" int iss_gather_halo_smem(int H, int W, int OH, int OW, int KH, int KW, int SH, int PT, int C, int N)
{
    if (C != HBK || KH * KW == 1) return 0;
    const int smem = halo_smem(f16_bn_for(N), iss_gather_halo_rows_bound(H, OH, OW, KH, SH, PT), W);
    return smem <= MAX_SMEM ? smem : 0;
}

int iss_gather_halo_rows(const ConvArgs &a)
{
    return iss_gather_halo_smem(a.H, a.W, a.OH, a.OW, a.KH, a.KW, a.SH, a.PT, a.C, a.N) ? iss_gather_halo_rows_bound(a.H, a.OH, a.OW, a.KH, a.SH, a.PT) : 0;
}

// Shared memory of a pooled gather-kernel layer (LD_POOL) on the pipelined path, 0 where it keeps another path: the layer
// takes the halo (64 input channels, more than one tap) and two halo buffers fit next to the three-stage weight ring.
extern "C" int iss_gather_pipe_smem(int H, int W, int OH, int OW, int KH, int KW, int SH, int PT, int C, int N)
{
    if (C != HBK || KH * KW == 1) return 0;
    const int smem = pipe_smem(f16_bn_for(N), iss_gather_halo_rows_bound(H, OH, OW, KH, SH, PT), W);
    return smem <= MAX_SMEM ? smem : 0;
}

int iss_gather_pipe_rows(const ConvArgs &a)
{
    return iss_gather_pipe_smem(a.H, a.W, a.OH, a.OW, a.KH, a.KW, a.SH, a.PT, a.C, a.N) ? iss_gather_halo_rows_bound(a.H, a.OH, a.OW, a.KH, a.SH, a.PT) : 0;
}

// Does the slab kernel take this engine-3 layer?  Un-padded, stride-1 'valid' convolution, 64 -> 64 channels, no
// folded pooling, and one slab plus a four-stage weight ring fit in shared memory.
bool iss_slab_covers(const ConvArgs &a)
{
    return a.C == SLAB_C && a.N == SLAB_N && a.K == a.KH * a.KW * a.C && a.pool_h == 0 &&
           a.SH == 1 && a.SW == 1 && a.PT == 0 && a.PL == 0 && a.OH == a.H - a.KH + 1 && a.OW == a.W - a.KW + 1 &&
           slab_smem(slab_rows(a.KH, a.KW, a.W), 1, SLAB_MAX_STAGES) <= SLAB_MAX_SMEM;
}

int iss_launch_conv_slab(const ConvArgs &a, cudaStream_t st)
{
    if (a.first) return launch_slab<LD_FIRST>(a, st);
    return a.in_packed ? launch_slab<LD_PACKED>(a, st) : launch_slab<LD_F32>(a, st);
}

int iss_launch_conv_f16(const ConvArgs &a, cudaStream_t st)
{
    return f16_bn_for(a.N) == 128 ? launch_f16<128>(a, st) : launch_f16<64>(a, st);
}

int iss_launch_conv_tf32(const ConvArgs &a, cudaStream_t st)
{
    switch (tf32_bn_for(a.N)) {
    case 128: return launch_wg<ENG_TF32, 128, LD_F32>(a, a.wt.tiled, 1.f, st);
    case 64: return launch_wg<ENG_TF32, 64, LD_F32>(a, a.wt.tiled, 1.f, st);
    default: return launch_wg<ENG_TF32, 32, LD_F32>(a, a.wt.tiled, 1.f, st);
    }
}

extern "C" int iss_set_gemm_mode(int mode)
{
    ISS_REQUIRE(mode == ISS_GEMM_FP32 || mode == ISS_GEMM_TC_TS || mode == ISS_GEMM_TC_F16, ISS_ERR_INVALID, "iss_set_gemm_mode: %d (0 = fp32 cores, 2 = 3xTF32, 3 = fp16 split)", mode);
    g_gemm_mode = mode;
    return ISS_OK;
}

extern "C" int iss_get_gemm_mode(void)
{
    if (g_gemm_mode < 0) {
        const char *e = getenv("ISS_B200_GEMM");
        g_gemm_mode = ISS_GEMM_DEFAULT;
        if (e && !strcmp(e, "fp32")) g_gemm_mode = ISS_GEMM_FP32;
        else if (e && !strcmp(e, "tc_ts")) g_gemm_mode = ISS_GEMM_TC_TS;
        else if (e && !strcmp(e, "tc_f16")) g_gemm_mode = ISS_GEMM_TC_F16;
    }
    return g_gemm_mode;
}

// Engine 2's image: [N/BN][K/32][hi | lo][BN rows x 32 floats], the 16-byte chunk j of row n stored at chunk j ^ (n & 7)
// (one cp.async stage per k-block).  Engine 3's: [N/BN][K/64][hi | lo][BN rows x 64 halves] in the same swizzle
// (f16_image.cuh), pre-scaled by a power of two.
int iss_prepare_weights(const float *h_w, int C, int K, int N, bool f16, TcWeights *w)
{
    *w = TcWeights{};
    if (C % 32 != 0 || K % 32 != 0 || N % 32 != 0) return ISS_OK;
    std::vector<float> wt((size_t)N * K);                         // transposed [N][K]
    for (int k = 0; k < K; ++k)
        for (int n = 0; n < N; ++n) wt[(size_t)n * K + k] = h_w[(size_t)k * N + n];
    const int BN = tf32_bn_for(N), nkb = K / TBK;
    std::vector<float> tiled((size_t)2 * N * K);
    for (int nt = 0; nt < N / BN; ++nt)
        for (int kb = 0; kb < nkb; ++kb) {
            float *hi = tiled.data() + ((size_t)nt * nkb + kb) * 2 * BN * TBK, *lo = hi + BN * TBK;
            for (int n = 0; n < BN; ++n)
                for (int k = 0; k < TBK; ++k) {
                    const float x = wt[(size_t)(nt * BN + n) * K + kb * TBK + k];
                    uint32_t u;
                    memcpy(&u, &x, 4);
                    u &= 0xFFFFE000u;
                    float h;
                    memcpy(&h, &u, 4);
                    const int o = n * TBK + (((k >> 2) ^ (n & 7)) << 2) + (k & 3);
                    hi[o] = h;
                    lo[o] = x - h;
                }
        }
    int rc = upload(tiled.data(), tiled.size() * sizeof(float), &w->tiled, "tc weights");
    if (rc != ISS_OK || !f16 || C % 64 != 0 || N % 64 != 0) return rc;
    std::vector<__half> img;
    const float scale = iss_f16_build_image(wt.data(), N, K, K, f16_bn_for(N), img);
    rc = upload(img.data(), img.size() * sizeof(__half), &w->f16, "f16 weights");
    if (rc == ISS_OK) w->f16_inv_scale = 1.f / scale;
    return rc;
}

void iss_free_weights(TcWeights *w)
{
    if (w->tiled) cudaFree(w->tiled);
    if (w->f16) cudaFree(w->f16);
    *w = TcWeights{};
}
