// conv_gemm.cu -- implicit-GEMM conv / dense on fp32 CUDA cores (see conv_gemm.cuh).
// 128 x {64,128} x 16 tiles, 8 x {4,8} register tiles, double-buffered shared memory,
// fused epilogue: bias -> BatchNorm affine -> (+residual) -> ReLU -> BatchNorm affine.
#include "conv_gemm.cuh"

namespace {

// ------------------------------------------------------------------ implicit-GEMM conv / dense (fp32 CUDA cores)
constexpr int BM = 128, BK = 16;

template <int BN, bool FIRST>
__global__ void __launch_bounds__(256, 2)
conv_gemm_f32_kernel(const ConvArgs a)
{
    constexpr int TM = 8, TN = BN / 16;
    __shared__ __align__(16) float As[2][BK][BM];
    __shared__ __align__(16) float Bs[2][BK][BN];
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    const int64_t m0 = (int64_t)blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;

    // ---- per-thread A-gather coordinates: one output position, 8 consecutive k per tile ----
    const int ml = tid & (BM - 1), kh2 = tid >> 7;
    const int64_t m = m0 + ml;
    const bool m_ok = m < a.M;
    int ih0 = 0, iw0 = 0;
    const float *in_img = a.in;
    float mu = 0.f, sg = 1.f;
    {
        const int64_t mm = m_ok ? m : 0;
        const int ohw = a.OH * a.OW;
        const int64_t img = mm / ohw;
        const int rem = (int)(mm - img * ohw);
        const int oh = rem / a.OW, ow = rem - oh * a.OW;
        ih0 = oh * a.SH - a.PT; iw0 = ow * a.SW - a.PL;
        if (FIRST) { in_img = a.in + (int64_t)a.row0[img] * a.ld; mu = a.mu[img]; sg = a.sigma[img]; }
        else in_img = a.in + img * ((int64_t)a.H * a.W * a.C);
    }
    const bool vecA = !FIRST && (a.C % 8 == 0);
    const bool vecB = (a.N % 4 == 0);

    float ra[8];
    float rb[TN];

    auto load_tiles = [&](int kt) {
        const int kb = kt * BK + kh2 * 8;
        if (vecA) {
            float4 v0 = make_float4(0.f, 0.f, 0.f, 0.f), v1 = v0;
            if (m_ok && kb < a.K) {
                const int tap = kb / a.C, c = kb - tap * a.C;
                const int r = tap / a.KW, s = tap - r * a.KW;
                const int ih = ih0 + r, iw = iw0 + s;
                if (ih >= 0 && ih < a.H && iw >= 0 && iw < a.W) {
                    const float4 *p = reinterpret_cast<const float4 *>(in_img + ((int64_t)ih * a.W + iw) * a.C + c);
                    v0 = __ldg(p); v1 = __ldg(p + 1);
                }
            }
            ra[0] = v0.x; ra[1] = v0.y; ra[2] = v0.z; ra[3] = v0.w;
            ra[4] = v1.x; ra[5] = v1.y; ra[6] = v1.z; ra[7] = v1.w;
        } else {
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const int k = kb + q;
                float v = 0.f;
                if (m_ok && k < a.K) {
                    const int tap = k / a.C, c = k - tap * a.C;
                    const int r = tap / a.KW, s = tap - r * a.KW;
                    const int ih = ih0 + r, iw = iw0 + s;
                    if (ih >= 0 && ih < a.H && iw >= 0 && iw < a.W) {
                        if (FIRST) v = __fdiv_rn(__fsub_rn(__ldg(in_img + (int64_t)ih * a.ld + iw), mu), sg);
                        else v = __ldg(in_img + ((int64_t)ih * a.W + iw) * a.C + c);
                    }
                }
                ra[q] = v;
            }
        }
        // B tile: BK x BN floats, 256 threads * TN
        {
            const int e = tid * TN;                  // element index in the tile
            const int kk = e / BN, nn = e - kk * BN;
            const int k = kt * BK + kk, n = n0 + nn;
            if (vecB && k < a.K && n + TN <= a.N) {
#pragma unroll
                for (int q = 0; q < TN; q += 4) {
                    const float4 v = __ldg(reinterpret_cast<const float4 *>(a.w + (int64_t)k * a.N + n + q));
                    rb[q] = v.x; rb[q + 1] = v.y; rb[q + 2] = v.z; rb[q + 3] = v.w;
                }
            } else {
#pragma unroll
                for (int q = 0; q < TN; ++q) rb[q] = (k < a.K && n + q < a.N) ? __ldg(a.w + (int64_t)k * a.N + n + q) : 0.f;
            }
        }
    };
    auto store_tiles = [&](int buf) {
#pragma unroll
        for (int q = 0; q < 8; ++q) As[buf][kh2 * 8 + q][ml] = ra[q];
        const int e = tid * TN;
        const int kk = e / BN, nn = e - kk * BN;
#pragma unroll
        for (int q = 0; q < TN; ++q) Bs[buf][kk][nn + q] = rb[q];
    };

    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    const int nkt = (a.K + BK - 1) / BK;
    load_tiles(0);
    store_tiles(0);
    __syncthreads();
    for (int kt = 0; kt < nkt; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < nkt) load_tiles(kt + 1);
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            float av[TM], bv[TN];
            const float4 a0 = *reinterpret_cast<const float4 *>(&As[buf][kk][ty * TM]);
            const float4 a1 = *reinterpret_cast<const float4 *>(&As[buf][kk][ty * TM + 4]);
            av[0] = a0.x; av[1] = a0.y; av[2] = a0.z; av[3] = a0.w; av[4] = a1.x; av[5] = a1.y; av[6] = a1.z; av[7] = a1.w;
#pragma unroll
            for (int q = 0; q < TN; q += 4) {
                const float4 b = *reinterpret_cast<const float4 *>(&Bs[buf][kk][tx * TN + q]);
                bv[q] = b.x; bv[q + 1] = b.y; bv[q + 2] = b.z; bv[q + 3] = b.w;
            }
#pragma unroll
            for (int i = 0; i < TM; ++i)
#pragma unroll
                for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        if (kt + 1 < nkt) store_tiles(buf ^ 1);
        __syncthreads();
    }

    // ---- epilogue ----
    EpiCoef1 cf[TN];
#pragma unroll
    for (int j = 0; j < TN; ++j) {
        const int n = n0 + tx * TN + j;
        if (n < a.N) cf[j] = epi_coef1(a, n);
    }
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const int64_t mr = m0 + ty * TM + i;
        if (mr >= a.M) continue;
        float v[TN];
#pragma unroll
        for (int j = 0; j < TN; ++j) {
            const int n = n0 + tx * TN + j;
            const float r = (a.flags & ISS_F_RESIDUAL) && n < a.N ? __ldg(a.residual + mr * a.N + n) : 0.f;
            v[j] = epi_f32<true>(cf[j], a.flags, acc[i][j], r);
        }
        float *o = a.out + mr * a.N + n0 + tx * TN;
        if (vecB && n0 + tx * TN + TN <= a.N) {
#pragma unroll
            for (int q = 0; q < TN; q += 4) *reinterpret_cast<float4 *>(o + q) = make_float4(v[q], v[q + 1], v[q + 2], v[q + 3]);
        } else {
#pragma unroll
            for (int j = 0; j < TN; ++j) if (n0 + tx * TN + j < a.N) o[j] = v[j];
        }
    }
}


// Dense / 1x1 layer with a handful of outputs (the softmax heads: 512 -> 2 or 3).  The generic 128 x 64 tile kernel spends
// 48 us on this 6 MFLOP layer (one column of CTAs, 3 useful columns of 64); here one warp owns a GEMM row, the K dimension
// is split over the lanes with 16-byte loads, the weights sit transposed [N][K] in shared memory (conflict-free float4
// reads) and the lane partials are combined in a fixed order (xor tree): deterministic, independent of the grid.
constexpr int SMALL_N = 8;
__global__ void __launch_bounds__(256)
dense_small_n_kernel(const ConvArgs a)
{
    extern __shared__ __align__(16) float wsm_t[];                 // [N][K]
    for (int i = threadIdx.x; i < a.K * a.N; i += 256) { const int k = i / a.N, n = i - k * a.N; wsm_t[n * a.K + k] = a.w[i]; }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int K4 = a.K >> 2;
    for (int64_t m = (int64_t)blockIdx.x * 8 + warp; m < a.M; m += (int64_t)gridDim.x * 8) {
        const float4 *x = reinterpret_cast<const float4 *>(a.in + m * a.K);
        float acc[SMALL_N];
#pragma unroll
        for (int n = 0; n < SMALL_N; ++n) acc[n] = 0.f;
        for (int k4 = lane; k4 < K4; k4 += 32) {
            const float4 v = __ldg(x + k4);
#pragma unroll
            for (int n = 0; n < SMALL_N; ++n) {
                if (n < a.N) {
                    const float4 w = *reinterpret_cast<const float4 *>(wsm_t + n * a.K + 4 * k4);
                    acc[n] = fmaf(v.x, w.x, acc[n]); acc[n] = fmaf(v.y, w.y, acc[n]);
                    acc[n] = fmaf(v.z, w.z, acc[n]); acc[n] = fmaf(v.w, w.w, acc[n]);
                }
            }
        }
#pragma unroll
        for (int n = 0; n < SMALL_N; ++n)
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) acc[n] += __shfl_xor_sync(0xffffffffu, acc[n], o);
        if (lane < a.N) {
            float xv = 0.f;
#pragma unroll
            for (int n = 0; n < SMALL_N; ++n) if (n == lane) xv = acc[n];
            a.out[m * a.N + lane] = epi_f32(epi_coef1(a, lane), a.flags, xv);
        }
    }
}

// ------------------------------------------------------------------ first layer: direct conv on the z-normalised patch
// The first Conv2D has one input channel (K = kh*kw ~ 20), far too thin for a GEMM tile.  One CTA
// stages a whole patch in shared memory, normalising each log-mel value exactly once with the
// reference's arithmetic ((x - mean) / std in float32, segmenter.py:82), zero-padded for 'same'
// convolutions; a thread owns 4 output channels x 4 consecutive output columns, so a filter tap is
// one LDS.128 (weights) + 4 broadcast LDS.32 (inputs) for 16 FMAs.  Taps are accumulated in the
// same (kh, kw) order as the implicit-GEMM kernel, so both produce identical bits.
constexpr int FIRST_P = 4;

// the zero-padded patch: H + PT + PB rows by W + PL + PR columns, for 'valid' and Keras 'same' padding alike
__host__ __device__ inline int first_hp(const ConvArgs &a) { return max(a.H + a.PT, (a.OH - 1) * a.SH + a.KH); }
__host__ __device__ inline int first_wp(const ConvArgs &a) { return max(a.W + a.PL, (a.OW - 1) * a.SW + a.KW); }

__global__ void __launch_bounds__(256)
conv_first_direct_kernel(const ConvArgs a)
{
    extern __shared__ __align__(16) float fsm[];
    const int Cout = a.N, Hp = first_hp(a), Wp = first_wp(a);
    float *ws = fsm;                                   // [K][Cout]
    float *xs = fsm + a.KH * a.KW * Cout;              // [Hp][Wp] (+ slack), zero border
    const int tid = threadIdx.x;
    const int CQ = Cout >> 2, streams = 256 / CQ;
    const int c4 = tid % CQ, stream = tid / CQ;
    const int K = a.KH * a.KW;
    for (int i = tid; i < K * Cout; i += 256) ws[i] = a.w[i];
    const int xs_len = Hp * Wp + FIRST_P * a.SW + a.KW;
    EpiCoef1 cf[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) cf[q] = epi_coef1(a, c4 * 4 + q);
    const int nblk = (a.OW + FIRST_P - 1) / FIRST_P;
    const int G = a.OH * nblk;
    const int64_t ohw = (int64_t)a.OH * a.OW;
    for (int64_t img = blockIdx.x; img * ohw < a.M; img += gridDim.x) {       // M / ohw patches
        __syncthreads();                               // previous patch fully consumed (and ws visible)
        for (int i = tid; i < xs_len; i += 256) xs[i] = 0.f;
        __syncthreads();
        const float mu = a.mu[img], sg = a.sigma[img];
        const float *src = a.in + (int64_t)a.row0[img] * a.ld;
        for (int e = tid; e < a.H * a.W; e += 256) {
            const int r = e / a.W, c = e - r * a.W;
            xs[(r + a.PT) * Wp + c + a.PL] = __fdiv_rn(__fsub_rn(__ldg(src + (int64_t)r * a.ld + c), mu), sg);
        }
        __syncthreads();
        float *out_img = a.out + img * ohw * Cout;
        for (int g = stream; g < G; g += streams) {
            const int oh = g / nblk, ow0 = (g - oh * nblk) * FIRST_P;
            float acc[FIRST_P][4];
#pragma unroll
            for (int p = 0; p < FIRST_P; ++p)
#pragma unroll
                for (int q = 0; q < 4; ++q) acc[p][q] = 0.f;
            for (int r = 0; r < a.KH; ++r) {
                const float *xrow = xs + (oh * a.SH + r) * Wp + ow0 * a.SW;
                const float *wrow = ws + (r * a.KW) * Cout + c4 * 4;
                for (int t = 0; t < a.KW; ++t) {
                    const float4 w4 = *reinterpret_cast<const float4 *>(wrow + t * Cout);
#pragma unroll
                    for (int p = 0; p < FIRST_P; ++p) {
                        const float x = xrow[p * a.SW + t];
                        acc[p][0] = fmaf(x, w4.x, acc[p][0]); acc[p][1] = fmaf(x, w4.y, acc[p][1]);
                        acc[p][2] = fmaf(x, w4.z, acc[p][2]); acc[p][3] = fmaf(x, w4.w, acc[p][3]);
                    }
                }
            }
#pragma unroll
            for (int p = 0; p < FIRST_P; ++p) {
                if (ow0 + p >= a.OW) continue;
                float y[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) y[q] = epi_f32(cf[q], a.flags, acc[p][q]);
                float *dst = out_img + ((int64_t)oh * a.OW + ow0 + p) * Cout + c4 * 4;
                if (a.out_packed)
                    *reinterpret_cast<uint4 *>(dst) = make_uint4(iss_pack_split(y[0]), iss_pack_split(y[1]), iss_pack_split(y[2]), iss_pack_split(y[3]));
                else
                    *reinterpret_cast<float4 *>(dst) = make_float4(y[0], y[1], y[2], y[3]);
            }
        }
    }
}

int launch_first_direct(const ConvArgs &a, cudaStream_t st)
{
    const size_t smem = ((size_t)a.KH * a.KW * a.N + (size_t)first_hp(a) * first_wp(a) + FIRST_P * a.SW + a.KW + 8) * sizeof(float);
    ISS_REQUIRE(smem <= 200 * 1024, ISS_ERR_UNSUPPORTED, "conv: first layer too large for the first-layer kernel");
    ISS_CUDA_OK(iss_optin_smem(reinterpret_cast<const void *>(conv_first_direct_kernel), 200 * 1024));
    int dev = 0, sms = 0;
    ISS_CUDA_OK(cudaGetDevice(&dev));
    ISS_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const int64_t n_img = a.M / ((int64_t)a.OH * a.OW);
    conv_first_direct_kernel<<<(unsigned)std::min<int64_t>(n_img, (int64_t)sms * 8), 256, smem, st>>>(a);
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch();
    return ISS_OK;
}

bool small_n_covers(const ConvArgs &a)
{
    return a.KH == 1 && a.KW == 1 && a.SH == 1 && a.SW == 1 && a.PT == 0 && a.PL == 0 && a.N <= SMALL_N && a.K % 4 == 0 && a.K == a.C &&
           (size_t)a.K * a.N * sizeof(float) <= 48 * 1024 && !a.in_packed && !a.out_packed && !(a.flags & ISS_F_RESIDUAL);
}

template <bool FIRST>
int launch_conv_t(const ConvArgs &a, cudaStream_t st)
{
    const int64_t gm = (a.M + BM - 1) / BM;
    ISS_REQUIRE(gm < (1ll << 31), ISS_ERR_INVALID, "conv: M too large");
    if (a.N <= 64) {
        dim3 grid((unsigned)gm, (unsigned)((a.N + 63) / 64));
        conv_gemm_f32_kernel<64, FIRST><<<grid, 256, 0, st>>>(a);
    } else {
        dim3 grid((unsigned)gm, (unsigned)((a.N + 127) / 128));
        conv_gemm_f32_kernel<128, FIRST><<<grid, 256, 0, st>>>(a);
    }
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch();
    return ISS_OK;
}

}  // namespace

IssConvKernel iss_conv_kernel(const ConvArgs &a, int mode)
{
    if (a.row0)
        return a.C == 1 && (a.N == 16 || a.N == 32 || a.N == 64 || a.N == 128) ? ISS_CONV_FIRST_DIRECT : ISS_CONV_F32_FIRST;
    if (small_n_covers(a)) return ISS_CONV_SMALL_N;
    if (mode == ISS_GEMM_FP32 || !a.wt.tiled || (a.flags & ISS_F_SIGMOID)) return ISS_CONV_F32;
    if (mode == ISS_GEMM_TC_F16 && a.wt.f16) {
        const bool slab = iss_slab_covers(a);
        // folded pooling: 2x2 / stride-2 'valid' over split-half words, in the gather kernel's operand fill
        const bool pool_ok = a.pool_h == 0 || (!a.first && a.in_packed && a.pool_h / 2 == a.H && a.pool_w / 2 == a.W);
        // the fused first layer: in the slab kernel's operand fill
        const bool first_ok = !a.first || (slab && !(a.flags & ISS_F_RESIDUAL));
        if (pool_ok && first_ok) return slab ? ISS_CONV_F16_SLAB : ISS_CONV_F16;
    }
    return ISS_CONV_TF32;
}

int iss_launch_conv(const ConvArgs &a, int mode, cudaStream_t st)
{
    const IssConvKernel k = iss_conv_kernel(a, mode);
    ISS_REQUIRE((iss_conv_is_f16(k) || (!a.in_packed && !a.residual_packed && !a.first && a.pool_h == 0)) &&
                (iss_conv_writes_words(k) || !a.out_packed), ISS_ERR_UNSUPPORTED,
                "conv: split-half tensors, folded pooling and the fused first layer need the fp16-split engine");
    switch (k) {
    case ISS_CONV_F32_FIRST: return launch_conv_t<true>(a, st);
    case ISS_CONV_FIRST_DIRECT: return launch_first_direct(a, st);
    case ISS_CONV_SMALL_N: {
        const int64_t gm = (a.M + 7) / 8;
        dense_small_n_kernel<<<(unsigned)(gm < 132 * 8 ? gm : 132 * 8), 256, (size_t)a.K * a.N * sizeof(float), st>>>(a);
        ISS_CUDA_OK(cudaGetLastError());
        iss_count_launch();
        return ISS_OK;
    }
    case ISS_CONV_TF32: return iss_launch_conv_tf32(a, st);
    case ISS_CONV_F16: return iss_launch_conv_f16(a, st);
    case ISS_CONV_F16_SLAB: return iss_launch_conv_slab(a, st);
    case ISS_CONV_F32: break;
    }
    return launch_conv_t<false>(a, st);
}
