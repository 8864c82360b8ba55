// feat_sidekit.cu -- K1: fused framing -> pre-emphasis -> log-energy -> Hann ->
// 512-point real FFT -> power -> 24-band mel -> log, one pass over the PCM.
//
// Reference semantics: inaSpeechSegmenter/sidekit_mfcc.py:200-237 (power_spectrum),
// :240-275 (framing, pre_emphasis), :118-197 (trfbank), :334 (log mel); only loge
// and mspec are produced because that is all segmenter.py:58 keeps.
//
// Layout: one CTA owns a tile of FR consecutive frames; the contiguous sample
// span of the tile ((FR-1)*160+400 samples, 2.5x frame overlap) is read from HBM
// exactly once with 16-byte vector loads and staged in shared memory together
// with the Hann window, the FFT twiddles and the sparse mel filterbank.  Each warp
// then processes frames independently: a 512-point real FFT is computed as a
// 256-point complex FFT held in registers (8 points per lane, ONE conflict-free
// transpose through shared memory + two rounds of shuffles: fft256r.cuh) followed
// by the even/odd split.  (Round 1 used a 4-pass radix-4 Stockham FFT through shared
// memory; with float64 data that was shared-memory bound: 33 % conflict wavefronts.)
// Round 2, second pass (the kernel was shared-memory bound at 580 wavefronts per frame): the even/odd split takes
// Z[256 - k] from its partner lane with register shuffles instead of a round trip of the spectrum through shared
// memory (partner lane / register algebra: tests/test_k1_split_model.py), the split twiddles are staged in lane order
// (conflict-free), and the 24 mel sums run as <= 32 balanced tasks (<= 24 bins each; a filter is up to three tasks)
// on all lanes instead of 24 lanes walking up to 48 bins.
// T = float: fast path; T = double: window/FFT/power in fp64 then rounded to f32,
// which is the reference's own precision recipe (sidekit_mfcc.py:231-233).
#include <math.h>
#include <string.h>
#include <type_traits>
#include <vector>

#include "iss_common.cuh"

namespace {

#include "fft256r.cuh"


constexpr int FR = 48;                               // frames per CTA tile (int16 staging + 48 frames => 3 CTAs/SM in fp64 mode)
constexpr int NWARP = 8;
constexpr int NTHREAD = NWARP * 32;
constexpr int TILE_SAMPLES = (FR - 1) * ISS_HOP + ISS_WIN;   // 7920
constexpr int ZPAD = 296;                            // power spectrum P[k] at k + 8 (k >> 6): 257 + 32, padded


template <typename T> struct Tab;
template <> struct Tab<float> {
    static __device__ __forceinline__ const float *win(const SidekitTables *t) { return t->win32; }
    static __device__ __forceinline__ const float *tw256(const SidekitTables *t) { return t->tw256_32; }
    static __device__ __forceinline__ const float *tw512(const SidekitTables *t) { return t->tw512_32; }
    static __device__ __forceinline__ float log_(float x) { return logf(x); }
};
template <> struct Tab<double> {
    static __device__ __forceinline__ const double *win(const SidekitTables *t) { return t->win64; }
    static __device__ __forceinline__ const double *tw256(const SidekitTables *t) { return t->tw256_64; }
    static __device__ __forceinline__ const double *tw512(const SidekitTables *t) { return t->tw512_64; }
    static __device__ __forceinline__ float log_(double x) { return (float)log(x); }
};

template <typename T, int PCM>
struct Smem {
    // staged verbatim: int16 PCM stays 2 bytes/sample in shared memory and is scaled by 1/32768 on use
    typename std::conditional<PCM == ISS_PCM_S16, int16_t, float>::type samples[TILE_SAMPLES + 8];
    T win[ISS_WIN];
    Cplx<T> twA[7 * 32];                    // W256^(lane * k1), k1 = 1..7 (fft256r.cuh)
    Cplx<T> twB[7 * 4];                     // W32^(r * k2a),   k2a = 1..7
    Cplx<T> twS[8 * 32];                    // W512^k of the bin lane l holds in register a, at [a * 32 + l] (split stage)
    float fbw[ISS_FB_MAXNNZ];
    int task_lo[32], task_cnt[32], task_off[32];      // mel tasks: bins [lo, lo + cnt) with weights fbw[off ..]
    int filt_first[ISS_NMEL], filt_n[ISS_NMEL];      // filter m = tasks [first, first + n)
    // per warp: the FFT's transpose rows; once the FFT is done the same bytes hold the power spectrum (ZPAD floats) and,
    // behind it, the per-task partial mel sums (32 T) -- keeps the CTA at 3 per SM (a separate pw / part array costs
    // 11 KB and drops it to 2)
    Cplx<T> buf[NWARP][FFT_BUF];
    double red[NWARP][2];
};
static_assert(ZPAD * sizeof(float) + 32 * sizeof(double) <= FFT_BUF * 2 * sizeof(float), "pw + part must fit the transpose buffer");

__device__ __forceinline__ int bitrev2(int r) { return ((r & 1) << 1) | ((r >> 1) & 1); }

// One recording of a features call.  Its tiles are [tile_off, next recording's tile_off); tile t starts at its frame
// FR * (t - tile_off), so a recording is tiled exactly as it would be on its own.
struct FeatRec {
    const void *pcm;
    int64_t n_frames;
    int64_t row_off;                // first mspec row
    int64_t loge_off;               // first loge entry
    int64_t tile_off;               // first tile (global block index); entry n_rec holds the total
    int vec_ok;                     // pcm is 16-byte aligned
};

template <typename T, int PCM>
__global__ void __launch_bounds__(NTHREAD, 3)
sidekit_features_kernel(const FeatRec *__restrict__ recs, int n_rec,
                        const SidekitTables *__restrict__ tabs, float *__restrict__ mspec_all,
                        float *__restrict__ loge_all, double *__restrict__ partials)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    Smem<T, PCM> &S = *reinterpret_cast<Smem<T, PCM> *>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);      // (a value the compiler knows to be warp-uniform: no re-convergence code around the frame loop's shuffles)
    int lo = 0, hi = n_rec;                                      // recs[lo].tile_off <= blockIdx.x < recs[hi].tile_off
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (recs[mid].tile_off <= (int64_t)blockIdx.x) lo = mid; else hi = mid; }
    const FeatRec &rec = recs[lo];
    const void *pcm = rec.pcm;
    const int64_t n_frames = rec.n_frames;
    const int vec_ok = rec.vec_ok;
    float *mspec = mspec_all + rec.row_off * ISS_NMEL;
    float *loge = loge_all + rec.loge_off;
    const int64_t f0 = ((int64_t)blockIdx.x - rec.tile_off) * FR;
    const int64_t s0 = f0 * ISS_HOP;
    const int nfr = (int)min((int64_t)FR, n_frames - f0);
    const int nsamp = (nfr - 1) * ISS_HOP + ISS_WIN;          // <= TILE_SAMPLES, all < n_samples

    // ---- stage tables (L2-resident, tiny) and the tile's samples (HBM, once) ----
    for (int i = tid; i < ISS_WIN; i += NTHREAD) S.win[i] = Tab<T>::win(tabs)[i];
    for (int i = tid; i < 7 * 32; i += NTHREAD) {                // W256^(l * k1) = tw256[l * k1]  (cos, -sin)
        const int k1 = i / 32 + 1, l = i % 32;
        S.twA[i].x = Tab<T>::tw256(tabs)[2 * (l * k1)]; S.twA[i].y = Tab<T>::tw256(tabs)[2 * (l * k1) + 1];
    }
    if (tid < 7 * 4) {                                           // W32^(r * k) = tw256[8 * r * k]
        const int k = tid / 4 + 1, r = tid % 4;
        S.twB[tid].x = Tab<T>::tw256(tabs)[2 * (8 * r * k)]; S.twB[tid].y = Tab<T>::tw256(tabs)[2 * (8 * r * k) + 1];
    }
    for (int i = tid; i < 8 * 32; i += NTHREAD) {                // lane l, register a holds bin (l >> 2) + 8 a + 64 bitrev2(l & 3)
        const int a = i >> 5, l = i & 31, k = (l >> 2) + 8 * a + 64 * bitrev2(l & 3);
        S.twS[i].x = Tab<T>::tw512(tabs)[2 * k]; S.twS[i].y = Tab<T>::tw512(tabs)[2 * k + 1];
    }
    for (int i = tid; i < tabs->nnz; i += NTHREAD) S.fbw[i] = tabs->w[i];
    if (tid < 32) { S.task_lo[tid] = tabs->task_lo[tid]; S.task_cnt[tid] = tabs->task_cnt[tid]; S.task_off[tid] = tabs->task_off[tid]; }
    if (tid < ISS_NMEL) { S.filt_first[tid] = tabs->filt_first[tid]; S.filt_n[tid] = tabs->filt_n[tid]; }

    if (PCM == ISS_PCM_S16) {
        const int16_t *p = reinterpret_cast<const int16_t *>(pcm) + s0;
        int16_t *dst = reinterpret_cast<int16_t *>(S.samples);
        if (vec_ok) {                                  // 8 samples per 16-byte load (tile offsets are multiples of 15360 B)
            const int nv = nsamp >> 3;
            const int4 *pv = reinterpret_cast<const int4 *>(p);
            int4 *dv = reinterpret_cast<int4 *>(dst);
            for (int i = tid; i < nv; i += NTHREAD) dv[i] = __ldg(pv + i);
            for (int i = (nv << 3) + tid; i < nsamp; i += NTHREAD) dst[i] = p[i];
        } else {
            for (int i = tid; i < nsamp; i += NTHREAD) dst[i] = p[i];
        }
    } else {
        const float *p = reinterpret_cast<const float *>(pcm) + s0;
        float *dst = reinterpret_cast<float *>(S.samples);
        if (vec_ok) {
            const int nv = nsamp >> 2;
            const float4 *pv = reinterpret_cast<const float4 *>(p);
            float4 *sv = reinterpret_cast<float4 *>(dst);
            for (int i = tid; i < nv; i += NTHREAD) sv[i] = __ldg(pv + i);
            for (int i = (nv << 2) + tid; i < nsamp; i += NTHREAD) dst[i] = p[i];
        } else {
            for (int i = tid; i < nsamp; i += NTHREAD) dst[i] = p[i];
        }
    }
    __syncthreads();

    Cplx<T> *buf = S.buf[warp];
    float *pw = reinterpret_cast<float *>(buf);                      // valid between the FFT's last __syncwarp and the next frame
    double acc_sum = 0.0, acc_cnt = 0.0;
    T *part = reinterpret_cast<T *>(reinterpret_cast<unsigned char *>(buf) + ZPAD * sizeof(float));
    // After the FFT this lane holds Z[k], k = zk1 + 8 a + 64 zk2b, in register a.  The split needs Z[256 - k]: it sits in
    // lane (8 - zk1) | (3 - r) at register 7 - a; for zk1 = 0 in lane 3 - r at register 8 - a, and for zk1 = 0, a = 0
    // (k = 0, 128, 64, 192) in lane {0, 1, 3, 2}[r].  Partners are always of the same class (zk1 = 0 or not), so the
    // SOURCE lane selects which register it sends.
    const int zk1 = lane >> 2, zr4 = lane & 3, zk2b = bitrev2(zr4);
    const bool cls0 = zk1 == 0;
    const int src_gen = cls0 ? (3 - zr4) : ((((8 - zk1) & 7) << 2) | (3 - zr4));
    const int src_a0 = cls0 ? (zr4 ^ (zr4 >> 1)) : src_gen;                      // {0, 1, 3, 2}[r]
    const int kbase = zk1 + 64 * zk2b;

    for (int fl = warp; fl < nfr; fl += NWARP) {
        const auto *xs = S.samples + fl * ISS_HOP;
        auto x = [&](int n) -> float {
            return (PCM == ISS_PCM_S16) ? (float)xs[n] * (1.0f / 32768.0f) : (float)xs[n];
        };
        // samples n, n + 1 (n even, the tile offset fl * 160 is even) in one load
        auto x2 = [&](int n, float &xa, float &xb) {
            if (PCM == ISS_PCM_S16) {
                const short2 v = *reinterpret_cast<const short2 *>(xs + n);
                xa = (float)v.x * (1.0f / 32768.0f); xb = (float)v.y * (1.0f / 32768.0f);
            } else {
                const float2 v = *reinterpret_cast<const float2 *>(xs + n);
                xa = v.x; xb = v.y;
            }
        };
        // ---- pre-emphasis (f32, numpy op order: x - (x_prev * 0.97f)), energy, window; the 512-point real
        //      frame is packed as z[m] = v[2m] + i v[2m+1] and lane l keeps z[32 n1 + l], n1 = 0..7, in registers ----
        T zr[8], zi[8];
        double e = 0.0;
#pragma unroll
        for (int n1 = 0; n1 < 8; ++n1) {
            const int n = 64 * n1 + 2 * lane;            // even sample of z[32 n1 + lane]; ISS_WIN is even
            T v0 = (T)0, v1 = (T)0;
            if (n < ISS_WIN) {
                float xa, xb;
                x2(n, xa, xb);
                const float xp = (n == 0) ? xa : x(n - 1);
                const float y0 = __fsub_rn(xa, __fmul_rn(xp, 0.97f));
                const float y1 = __fsub_rn(xb, __fmul_rn(xa, 0.97f));
                e += (double)y0 * (double)y0;
                e += (double)y1 * (double)y1;
                v0 = (T)y0 * S.win[n];
                v1 = (T)y1 * S.win[n + 1];
            }
            zr[n1] = v0; zi[n1] = v1;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) e += __shfl_xor_sync(0xffffffffu, e, o);

        warp_fft256_reg<T>(zr, zi, buf, S.twA, S.twB, lane);

        // ---- even/odd split X[k] = E[k] + W512^k O[k] with Z[256 - k] from the partner lane (shuffles), power -> f32 at
        //      pw[k + 8 (k >> 6)] (conflict-free: the 32 lanes' bins of one register cover all banks) ----
#pragma unroll
        for (int a = 0; a < 8; ++a) {
            const T sr = cls0 ? zr[(8 - a) & 7] : zr[7 - a], si = cls0 ? zi[(8 - a) & 7] : zi[7 - a];
            const int src = (a == 0) ? src_a0 : src_gen;
            const T cr = __shfl_sync(0xffffffffu, sr, src), ci = -__shfl_sync(0xffffffffu, si, src);      // conj(Z[256-k])
            const T zr_ = zr[a], zi_ = zi[a];
            const T er = (T)0.5 * (zr_ + cr), ei = (T)0.5 * (zi_ + ci);
            const T dr = (T)0.5 * (zr_ - cr), di = (T)0.5 * (zi_ - ci);
            const T orr = di, oi = -dr;                              // O = -i * (Z - conj)/2
            const Cplx<T> w = S.twS[a * 32 + lane];
            const T xr = er + (orr * w.x - oi * w.y);
            const T xi = ei + (orr * w.y + oi * w.x);
            const int k = kbase + 8 * a;
            pw[k + 8 * (k >> 6)] = (float)(xr * xr + xi * xi);
            if (a == 0 && lane == 0) {                               // k = 0 also yields the Nyquist bin: X[256] = Re Z[0] - Im Z[0]
                const T xn = zr_ - zi_;
                pw[256 + 8 * 4] = (float)(xn * xn);
            }
        }
        __syncwarp();

        // ---- mel filterbank (sparse triangles) as balanced tasks on all lanes, then <= 3 partials per filter + log ----
        const int64_t f = f0 + fl;
        {
            const int lo = S.task_lo[lane], cnt = S.task_cnt[lane];
            const float *w = S.fbw + S.task_off[lane];
            T acc0 = (T)0, acc1 = (T)0;                              // two chains: the kernel is latency-bound
            int b = 0;
            for (; b + 1 < cnt; b += 2) {
                const int k = lo + b, k2 = k + 1;
                acc0 += (T)pw[k + 8 * (k >> 6)] * (T)w[b];
                acc1 += (T)pw[k2 + 8 * (k2 >> 6)] * (T)w[b + 1];
            }
            if (b < cnt) { const int k = lo + b; acc0 += (T)pw[k + 8 * (k >> 6)] * (T)w[b]; }
            part[lane] = acc0 + acc1;
        }
        __syncwarp();
        if (lane < ISS_NMEL) {
            const int t0 = S.filt_first[lane], tn = S.filt_n[lane];
            T acc = (T)0;
            for (int t = 0; t < tn; ++t) acc += part[t0 + t];
            mspec[f * ISS_NMEL + lane] = Tab<T>::log_((T)(float)acc);
        }
        const float le = Tab<T>::log_((T)(float)e);
        if (lane == 0) {
            loge[f] = le;
            if (isfinite(le)) { acc_sum += (double)le; acc_cnt += 1.0; }
        }
        __syncwarp();
    }

    // ---- per-tile partial of {sum, count} of finite loge: fixed order, no atomics ----
    if (lane == 0) { S.red[warp][0] = acc_sum; S.red[warp][1] = acc_cnt; }
    __syncthreads();
    if (tid == 0) {
        double s = 0.0, c = 0.0;
#pragma unroll
        for (int w = 0; w < NWARP; ++w) { s += S.red[w][0]; c += S.red[w][1]; }
        partials[2 * (int64_t)blockIdx.x] = s;
        partials[2 * (int64_t)blockIdx.x + 1] = c;
    }
}

// Block b reduces the tiles of recording b (recs == nullptr: the single sequence of ntiles tiles) into stats[b][2];
// the order depends only on the tile's index within its recording, so a recording gives the same bits in any call.
__global__ void __launch_bounds__(1024, 1)
loge_stats_finalize_kernel(const double *__restrict__ partials, const FeatRec *__restrict__ recs, int64_t ntiles,
                           double *__restrict__ stats)
{
    __shared__ double ss[1024], sc[1024];
    if (recs) {
        partials += 2 * recs[blockIdx.x].tile_off;
        ntiles = recs[blockIdx.x + 1].tile_off - recs[blockIdx.x].tile_off;
        stats += 2 * blockIdx.x;
    }
    double s = 0.0, c = 0.0;
    for (int64_t i = threadIdx.x; i < ntiles; i += 1024) { s += partials[2 * i]; c += partials[2 * i + 1]; }
    ss[threadIdx.x] = s; sc[threadIdx.x] = c;
    __syncthreads();
    for (int o = 512; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) { ss[threadIdx.x] += ss[threadIdx.x + o]; sc[threadIdx.x] += sc[threadIdx.x + o]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { stats[0] = ss[0]; stats[1] = sc[0]; }
}

// Same arithmetic as the fused per-tile partials above: warp w of a tile sums the
// frames w, w+8, ... in order, the tile sums its 8 warps in order.
__device__ __forceinline__ void loge_tile_partial(const float *__restrict__ loge, int64_t L, int64_t tile,
                                                  double *__restrict__ partials)
{
    const int64_t f0 = tile * FR;
    const int nfr = (int)min((int64_t)FR, L - f0);
    double s = 0.0, c = 0.0;
    for (int w = 0; w < NWARP; ++w) {
        double sw = 0.0, cw = 0.0;
        for (int fl = w; fl < nfr; fl += NWARP) {
            const float le = loge[f0 + fl];
            if (isfinite(le)) { sw += (double)le; cw += 1.0; }
        }
        s += sw; c += cw;
    }
    partials[0] = s;
    partials[1] = c;
}

__global__ void __launch_bounds__(128)
loge_tile_partials_kernel(const float *__restrict__ loge, int64_t L, int64_t ntiles, double *__restrict__ partials)
{
    const int64_t tile = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tile >= ntiles) return;
    loge_tile_partial(loge, L, tile, partials + 2 * tile);
}

// The tiles of many sequences (recording r: loge_off / n_frames / tile_off of recs[r]), each tiled from its own start.
__global__ void __launch_bounds__(128)
loge_tile_partials_multi_kernel(const float *__restrict__ loge, const FeatRec *__restrict__ recs, int n_rec,
                                int64_t ntiles, double *__restrict__ partials)
{
    const int64_t tile = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tile >= ntiles) return;
    int lo = 0, hi = n_rec;                            // recs[lo].tile_off <= tile < recs[hi].tile_off
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (recs[mid].tile_off <= tile) lo = mid; else hi = mid; }
    const FeatRec r = recs[lo];
    loge_tile_partial(loge + r.loge_off, r.n_frames, tile - r.tile_off, partials + 2 * tile);
}

}  // namespace

static int ensure_partials(iss_ctx *ctx, int64_t ntiles)
{
    if (ntiles > ctx->partials_cap) {
        if (ctx->d_partials) ISS_CUDA_OK(cudaFree(ctx->d_partials));
        ctx->d_partials = nullptr; ctx->partials_cap = 0;
        const int64_t cap = ntiles + ntiles / 2 + 1024;
        cudaError_t e = cudaMalloc(&ctx->d_partials, (size_t)cap * 2 * sizeof(double));
        if (e != cudaSuccess) { iss_set_error("cudaMalloc partials: %s", cudaGetErrorString(e)); return ISS_ERR_NOMEM; }
        ctx->partials_cap = cap;
    }
    return ISS_OK;
}

static int ensure_recs(iss_ctx *ctx, int n_rec)
{
    if (n_rec + 1 > ctx->recs_cap) {
        if (ctx->d_recs) ISS_CUDA_OK(cudaFree(ctx->d_recs));
        ctx->d_recs = nullptr; ctx->recs_cap = 0;
        const int64_t cap = n_rec + 1 + n_rec / 2 + 64;
        cudaError_t e = cudaMalloc(&ctx->d_recs, (size_t)cap * sizeof(FeatRec));
        if (e != cudaSuccess) { iss_set_error("cudaMalloc recording table: %s", cudaGetErrorString(e)); return ISS_ERR_NOMEM; }
        ctx->recs_cap = cap;
    }
    return ISS_OK;
}

extern "C" int iss_loge_stats(iss_ctx *ctx, const float *d_loge, int64_t L, double *d_loge_stats, void *stream)
{
    ISS_REQUIRE(ctx && d_loge_stats, ISS_ERR_INVALID, "iss_loge_stats: NULL argument");
    ISS_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = iss_stream(stream);
    if (L <= 0) { ISS_CUDA_OK(cudaMemsetAsync(d_loge_stats, 0, 2 * sizeof(double), st)); return ISS_OK; }
    ISS_REQUIRE(d_loge, ISS_ERR_INVALID, "iss_loge_stats: NULL buffer");
    const int64_t ntiles = (L + FR - 1) / FR;
    int rc = ensure_partials(ctx, ntiles);
    if (rc != ISS_OK) return rc;
    loge_tile_partials_kernel<<<(unsigned)((ntiles + 127) / 128), 128, 0, st>>>(d_loge, L, ntiles, ctx->d_partials);
    loge_stats_finalize_kernel<<<1, 1024, 0, st>>>(ctx->d_partials, nullptr, ntiles, d_loge_stats);
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch(2);
    return ISS_OK;
}

extern "C" int64_t iss_sidekit_num_frames(int64_t n_samples)
{
    if (n_samples < ISS_WIN) return 0;
    return (n_samples - ISS_WIN) / ISS_HOP + 1;
}

extern "C" int iss_sidekit_upload_tables(iss_ctx *ctx, const float *h_fbank, const double *h_window)
{
    ISS_REQUIRE(ctx && h_fbank && h_window, ISS_ERR_INVALID, "iss_sidekit_upload_tables: NULL argument");
    ISS_CUDA_OK(cudaSetDevice(ctx->device));
    SidekitTables *t = new SidekitTables();
    memset(t, 0, sizeof(*t));
    int nnz = 0;
    for (int m = 0; m < ISS_NMEL; ++m) {
        int lo = -1, hi = -1;
        for (int k = 0; k < ISS_NBIN; ++k)
            if (h_fbank[m * ISS_NBIN + k] != 0.0f) { if (lo < 0) lo = k; hi = k; }
        t->lo[m] = lo < 0 ? 0 : lo;
        t->cnt[m] = lo < 0 ? 0 : hi - lo + 1;
        t->off[m] = nnz;
        if (nnz + t->cnt[m] > ISS_FB_MAXNNZ) {
            delete t;
            iss_set_error("iss_sidekit_upload_tables: filterbank support too wide");
            return ISS_ERR_INVALID;
        }
        for (int b = 0; b < t->cnt[m]; ++b) t->w[nnz++] = h_fbank[m * ISS_NBIN + lo + b];
    }
    t->nnz = nnz;
    {   // balanced mel tasks: the smallest cap (bins per task) for which all filters fit 32 tasks; a filter's bins are
        // dealt to its tasks as evenly as possible
        int cap = 1;
        for (;; ++cap) {
            int n = 0;
            for (int m = 0; m < ISS_NMEL; ++m) n += (t->cnt[m] + cap - 1) / cap;
            if (n <= 32) break;
        }
        int nt = 0;
        for (int m = 0; m < ISS_NMEL; ++m) {
            const int parts = (t->cnt[m] + cap - 1) / cap;
            t->filt_first[m] = nt; t->filt_n[m] = parts;
            int done = 0;
            for (int q = 0; q < parts; ++q) {
                const int len = (t->cnt[m] - done + (parts - q) - 1) / (parts - q);
                t->task_lo[nt] = t->lo[m] + done; t->task_cnt[nt] = len; t->task_off[nt] = t->off[m] + done;
                done += len; ++nt;
            }
        }
        for (; nt < 32; ++nt) { t->task_lo[nt] = 0; t->task_cnt[nt] = 0; t->task_off[nt] = 0; }
    }
    const double PI = 3.14159265358979323846;
    for (int i = 0; i < ISS_WIN; ++i) { t->win64[i] = h_window[i]; t->win32[i] = (float)h_window[i]; }
    for (int m = 0; m < 256; ++m) {
        const double c = cos(2.0 * PI * m / 256.0), s = -sin(2.0 * PI * m / 256.0);
        t->tw256_64[2 * m] = c; t->tw256_64[2 * m + 1] = s;
        t->tw256_32[2 * m] = (float)c; t->tw256_32[2 * m + 1] = (float)s;
    }
    for (int k = 0; k <= 256; ++k) {
        const double c = cos(2.0 * PI * k / 512.0), s = -sin(2.0 * PI * k / 512.0);
        t->tw512_64[2 * k] = c; t->tw512_64[2 * k + 1] = s;
        t->tw512_32[2 * k] = (float)c; t->tw512_32[2 * k + 1] = (float)s;
    }
    if (!ctx->d_tables) {
        cudaError_t e = cudaMalloc(&ctx->d_tables, sizeof(SidekitTables));
        if (e != cudaSuccess) { delete t; iss_set_error("cudaMalloc tables: %s", cudaGetErrorString(e)); return ISS_ERR_NOMEM; }
    }
    cudaError_t e = cudaMemcpy(ctx->d_tables, t, sizeof(SidekitTables), cudaMemcpyHostToDevice);
    delete t;
    if (e != cudaSuccess) { iss_set_error("cudaMemcpy tables: %s", cudaGetErrorString(e)); return ISS_ERR_CUDA; }
    ctx->tables_ready = true;
    return ISS_OK;
}

template <typename T, int PCM>
static int launch_features(iss_ctx *ctx, const FeatRec *d_recs, int n_rec, int64_t ntiles, float *d_mspec, float *d_loge,
                           cudaStream_t st)
{
    auto kern = sidekit_features_kernel<T, PCM>;
    const size_t smem = sizeof(Smem<T, PCM>);
    ISS_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<(unsigned)ntiles, NTHREAD, smem, st>>>(d_recs, n_rec, ctx->d_tables, d_mspec, d_loge, ctx->d_partials);
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch();
    return ISS_OK;
}

extern "C" int iss_sidekit_features_multi(iss_ctx *ctx, int n_rec, const void *const *h_pcm, const int64_t *h_n_samples,
                                          int pcm_format, int fft_precision, float *d_mspec, const int64_t *h_row_off,
                                          float *d_loge, const int64_t *h_loge_off, double *d_loge_stats, void *stream)
{
    ISS_REQUIRE(ctx, ISS_ERR_INVALID, "iss_sidekit_features: ctx is NULL");
    ISS_REQUIRE(ctx->tables_ready, ISS_ERR_STATE, "iss_sidekit_features: call iss_sidekit_upload_tables first");
    ISS_REQUIRE(pcm_format == ISS_PCM_F32 || pcm_format == ISS_PCM_S16, ISS_ERR_INVALID, "bad pcm_format %d", pcm_format);
    ISS_REQUIRE(fft_precision == ISS_FFT_FP32 || fft_precision == ISS_FFT_FP64, ISS_ERR_INVALID, "bad fft_precision %d", fft_precision);
    ISS_REQUIRE(n_rec >= 1 && h_pcm && h_n_samples && h_row_off && h_loge_off, ISS_ERR_INVALID, "iss_sidekit_features_multi: bad argument");
    ISS_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = iss_stream(stream);
    std::vector<FeatRec> recs(n_rec + 1);
    int64_t ntiles = 0;
    for (int i = 0; i < n_rec; ++i) {
        FeatRec &r = recs[i];
        r.pcm = h_pcm[i];
        r.n_frames = iss_sidekit_num_frames(h_n_samples[i]);
        r.row_off = h_row_off[i]; r.loge_off = h_loge_off[i]; r.tile_off = ntiles;
        r.vec_ok = ((reinterpret_cast<uintptr_t>(r.pcm) & 15) == 0) ? 1 : 0;
        ISS_REQUIRE(r.n_frames == 0 || r.pcm, ISS_ERR_INVALID, "iss_sidekit_features: NULL buffer (recording %d)", i);
        ISS_REQUIRE(r.row_off >= 0 && r.loge_off >= 0, ISS_ERR_INVALID, "iss_sidekit_features_multi: negative offset (recording %d)", i);
        ntiles += (r.n_frames + FR - 1) / FR;
    }
    recs[n_rec] = FeatRec{nullptr, 0, 0, 0, ntiles, 0};
    if (ntiles == 0) {
        if (d_loge_stats) ISS_CUDA_OK(cudaMemsetAsync(d_loge_stats, 0, 2 * sizeof(double) * n_rec, st));
        return ISS_OK;
    }
    ISS_REQUIRE(d_mspec && d_loge, ISS_ERR_INVALID, "iss_sidekit_features: NULL buffer");
    ISS_REQUIRE(ntiles < (1ll << 31), ISS_ERR_INVALID, "iss_sidekit_features: signal too long for one call");
    {
        const int prc = ensure_partials(ctx, ntiles);
        if (prc != ISS_OK) return prc;
    }
    {
        const int rrc = ensure_recs(ctx, n_rec);
        if (rrc != ISS_OK) return rrc;
    }
    const FeatRec *d_recs = reinterpret_cast<const FeatRec *>(ctx->d_recs);
    ISS_CUDA_OK(cudaMemcpyAsync(ctx->d_recs, recs.data(), sizeof(FeatRec) * (n_rec + 1), cudaMemcpyHostToDevice, st));
    int rc;
    if (fft_precision == ISS_FFT_FP32)
        rc = (pcm_format == ISS_PCM_S16)
                 ? launch_features<float, ISS_PCM_S16>(ctx, d_recs, n_rec, ntiles, d_mspec, d_loge, st)
                 : launch_features<float, ISS_PCM_F32>(ctx, d_recs, n_rec, ntiles, d_mspec, d_loge, st);
    else
        rc = (pcm_format == ISS_PCM_S16)
                 ? launch_features<double, ISS_PCM_S16>(ctx, d_recs, n_rec, ntiles, d_mspec, d_loge, st)
                 : launch_features<double, ISS_PCM_F32>(ctx, d_recs, n_rec, ntiles, d_mspec, d_loge, st);
    if (rc != ISS_OK) return rc;
    if (d_loge_stats) {
        loge_stats_finalize_kernel<<<(unsigned)n_rec, 1024, 0, st>>>(ctx->d_partials, d_recs, 0, d_loge_stats);
        ISS_CUDA_OK(cudaGetLastError());
        iss_count_launch();
    }
    return ISS_OK;
}

extern "C" int iss_sidekit_features(iss_ctx *ctx, const void *d_pcm, int pcm_format, int64_t n_samples,
                                    int fft_precision, float *d_mspec, float *d_loge,
                                    double *d_loge_stats, void *stream)
{
    const int64_t zero = 0;
    return iss_sidekit_features_multi(ctx, 1, &d_pcm, &n_samples, pcm_format, fft_precision, d_mspec, &zero, d_loge, &zero,
                                      d_loge_stats, stream);
}

extern "C" int iss_loge_stats_multi(iss_ctx *ctx, const float *d_loge, const int64_t *h_loge_off, const int64_t *h_len,
                                    int n_seq, double *d_loge_stats, void *stream)
{
    ISS_REQUIRE(ctx && d_loge_stats && h_loge_off && h_len && n_seq >= 1, ISS_ERR_INVALID, "iss_loge_stats_multi: bad argument");
    ISS_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = iss_stream(stream);
    std::vector<FeatRec> recs(n_seq + 1);
    int64_t ntiles = 0;
    for (int i = 0; i < n_seq; ++i) {
        ISS_REQUIRE(h_len[i] >= 1 && h_loge_off[i] >= 0, ISS_ERR_INVALID, "iss_loge_stats_multi: sequence %d is empty", i);
        recs[i] = FeatRec{nullptr, h_len[i], 0, h_loge_off[i], ntiles, 0};
        ntiles += (h_len[i] + FR - 1) / FR;
    }
    recs[n_seq] = FeatRec{nullptr, 0, 0, 0, ntiles, 0};
    ISS_REQUIRE(d_loge, ISS_ERR_INVALID, "iss_loge_stats_multi: NULL buffer");
    int rc = ensure_partials(ctx, ntiles);
    if (rc != ISS_OK) return rc;
    rc = ensure_recs(ctx, n_seq);
    if (rc != ISS_OK) return rc;
    FeatRec *d_recs = reinterpret_cast<FeatRec *>(ctx->d_recs);
    ISS_CUDA_OK(cudaMemcpyAsync(d_recs, recs.data(), sizeof(FeatRec) * (n_seq + 1), cudaMemcpyHostToDevice, st));
    loge_tile_partials_multi_kernel<<<(unsigned)((ntiles + 127) / 128), 128, 0, st>>>(d_loge, d_recs, n_seq, ntiles,
                                                                                      ctx->d_partials);
    loge_stats_finalize_kernel<<<(unsigned)n_seq, 1024, 0, st>>>(ctx->d_partials, d_recs, 0, d_loge_stats);
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch(2);
    return ISS_OK;
}
