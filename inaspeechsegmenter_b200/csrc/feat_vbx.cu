// feat_vbx.cu -- K4: VBx / HTK-style 64-band log-mel front-end + floating CMVN.
//
// Reference semantics: get_features (inaSpeechSegmenter/vbx_segmenter.py:72-89):
//   x = trunc(signal * 2^15) + dither              (:85, features_vbx.py:127-128)
//   mirror pad 120 left / 200 right                 (:86)
//   fbank_htk(..., USEPOWER=True, ZMEANSOURCE=True) (features_vbx.py:62-120): frames
//   400/160, per-frame mean removal (:100-101), per-frame pre-emphasis 0.97 (:104-105),
//   Povey window (:123-124), rfft 512, power, log(max(1, P . fbank)) (:109-113)
//   cmvn_floating_kaldi(fea, 150, 149, norm_vars=False) (:131-148), cast to float32.
// Everything is float64 like the reference.  The dither is a prefix of ONE fixed
// MT19937 sequence (np.random.seed(3)), so it is an input stream (device-resident
// cache owned by the host side), not something to regenerate per call.
//
// Kernel A: tile of FR frames per CTA, padded/dithered samples staged once in shared
// memory as doubles, one frame per warp iteration, FFT from fft256.cuh, sparse 64-band
// filterbank, raw log-fbank written as float64 [M][64] to scratch.
// Kernel B: sliding 300-frame mean (Kaldi edge handling: the window shifts, it does
// not shrink), one thread per band, 128-frame chunks: direct sum for the first frame
// of the chunk, then add/subtract one row per step.
// Both kernels take a table of recordings (iss_vbx_features_multi): a CTA finds its
// recording by binary search over the tile / chunk offsets, and every index inside it
// (padding, dither, tile, CMVN window) is local to that recording.
#include <math.h>
#include <string.h>
#include <vector>

#include "iss_common.cuh"

namespace {

#include "fft256.cuh"

constexpr int VFR = 16;                                 // frames per CTA tile (2 CTAs/SM at ~94 KB smem)
constexpr int VNWARP = 8;
constexpr int VNTHREAD = VNWARP * 32;
constexpr int VTILE = (VFR - 1) * ISS_HOP + ISS_WIN;    // 2800 samples
constexpr int VZPAD = 272;
constexpr int VBANDS = 64;
constexpr int VMAXNNZ = 1024;
constexpr int VPADL = 120, VPADR = 200;                 // noverlap/2, winlen/2 (vbx_segmenter.py:86)
constexpr int CMVN_LC = 150, CMVN_WIN = 300;
constexpr int CMVN_CHUNK = 128;

}  // namespace

struct VbxTables {
    int lo[VBANDS], cnt[VBANDS], off[VBANDS];
    int nnz;
    double w[VMAXNNZ];
    double win[ISS_WIN];
    double tw256[512];
    double tw512[2 * 257 + 2];
};

namespace {

struct VSmem {
    double samples[VTILE];
    double win[ISS_WIN];
    double tw256[512];
    double tw512[2 * 257 + 2];
    double fbw[VMAXNNZ];
    int fb_lo[VBANDS], fb_cnt[VBANDS], fb_off[VBANDS];
    double re[VNWARP][VZPAD];
    double im[VNWARP][VZPAD];
    double pw[VNWARP][VZPAD];
};

template <int PCM>
__device__ __forceinline__ double load_quantised(const void *pcm, int64_t i)
{
    // (signal * 2**15).astype(int): int16 PCM is already that integer; float input is truncated toward zero
    if (PCM == ISS_PCM_S16) return (double)reinterpret_cast<const int16_t *>(pcm)[i];
    return trunc((double)reinterpret_cast<const float *>(pcm)[i] * 32768.0);
}

// One recording of a features call.  Its fbank tiles are [tile_off, next recording's tile_off) and its CMVN chunks
// [chunk_off, next chunk_off); tile t starts at its frame VFR * (t - tile_off) and chunk c at CMVN_CHUNK * (c - chunk_off),
// so a recording is tiled, padded, dithered and normalised exactly as it would be on its own.
struct VbxRec {
    const void *pcm;
    int64_t n;                      // samples
    int64_t M;                      // feature frames
    int64_t raw_off;                // first row of the float64 scratch
    int64_t fea_off;                // first output row
    int64_t tile_off;               // first fbank tile (global block index); entry n_rec holds the total
    int64_t chunk_off;              // first CMVN chunk (global block index); entry n_rec holds the total
};

// recs[lo].off <= b < recs[hi].off (recordings without frames own no block)
template <int64_t VbxRec::*OFF>
__device__ __forceinline__ const VbxRec &find_rec(const VbxRec *__restrict__ recs, int n_rec, int64_t b)
{
    int lo = 0, hi = n_rec;
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (recs[mid].*OFF <= b) lo = mid; else hi = mid; }
    return recs[lo];
}

template <int PCM>
__global__ void __launch_bounds__(VNTHREAD, 2)
vbx_fbank_kernel(const VbxRec *__restrict__ recs, int n_rec, const double *__restrict__ dither,
                 const VbxTables *__restrict__ tabs, double *__restrict__ raw_all)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    VSmem &S = *reinterpret_cast<VSmem *>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const VbxRec &rec = find_rec<&VbxRec::tile_off>(recs, n_rec, blockIdx.x);
    const void *pcm = rec.pcm;
    const int64_t n = rec.n, M = rec.M;
    double *raw = raw_all + rec.raw_off * VBANDS;
    const int64_t f0 = ((int64_t)blockIdx.x - rec.tile_off) * VFR;
    const int nfr = (int)min((int64_t)VFR, M - f0);
    const int nsamp = (nfr - 1) * ISS_HOP + ISS_WIN;
    const int64_t p0 = f0 * ISS_HOP;                    // first index in the mirror-padded signal

    for (int i = tid; i < ISS_WIN; i += VNTHREAD) S.win[i] = tabs->win[i];
    for (int i = tid; i < 512; i += VNTHREAD) S.tw256[i] = tabs->tw256[i];
    for (int i = tid; i < 2 * 257; i += VNTHREAD) S.tw512[i] = tabs->tw512[i];
    for (int i = tid; i < tabs->nnz; i += VNTHREAD) S.fbw[i] = tabs->w[i];
    if (tid < VBANDS) { S.fb_lo[tid] = tabs->lo[tid]; S.fb_cnt[tid] = tabs->cnt[tid]; S.fb_off[tid] = tabs->off[tid]; }
    for (int i = tid; i < nsamp; i += VNTHREAD) {
        const int64_t p = p0 + i;                       // padded index in [0, n + 320)
        int64_t src;
        if (p < VPADL) src = VPADL - 1 - p;             // signal[119::-1]
        else if (p < VPADL + n) src = p - VPADL;
        else src = 2 * n + VPADL - 1 - p;               // signal[-1:-201:-1]
        double v = load_quantised<PCM>(pcm, src);
        if (dither) v += dither[src];
        S.samples[i] = v;
    }
    __syncthreads();

    double *re = S.re[warp], *im = S.im[warp], *pw = S.pw[warp];
    for (int fl = warp; fl < nfr; fl += VNWARP) {
        const double *x = S.samples + fl * ISS_HOP;
        // frame mean (ZMEANSOURCE)
        double s = 0.0;
#pragma unroll
        for (int i = 0; i < 13; ++i) { const int k = lane + 32 * i; if (k < ISS_WIN) s += x[k]; }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        const double mean = s / (double)ISS_WIN;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const int k = lane + 32 * i;
            double v = 0.0;
            if (k < ISS_WIN) {
                const double xc = x[k] - mean;
                const double xp = (k == 0) ? xc : (x[k - 1] - mean);
                v = __dsub_rn(xc, __dmul_rn(xp, 0.97)) * S.win[k];
            }
            if (k & 1) im[skewT<double>(k >> 1)] = v; else re[skewT<double>(k >> 1)] = v;
        }
        __syncwarp();
        warp_fft256<double>(re, im, S.tw256, lane);
#pragma unroll
        for (int i = 0; i < 9; ++i) {
            const int k = lane + 32 * i;
            if (k <= 256) {
                const int ka = skewT<double>(k & 255), kb = skewT<double>((256 - k) & 255);
                const double zr = re[ka], zi = im[ka];
                const double cr = re[kb], ci = -im[kb];
                const double er = 0.5 * (zr + cr), ei = 0.5 * (zi + ci);
                const double dr = 0.5 * (zr - cr), di = 0.5 * (zi - ci);
                const double orr = di, oi = -dr;
                const double c = S.tw512[2 * k], sn = S.tw512[2 * k + 1];
                const double xr = er + (orr * c - oi * sn);
                const double xi = ei + (orr * sn + oi * c);
                pw[k + (k >> 5)] = xr * xr + xi * xi;
            }
        }
        __syncwarp();
        const int64_t f = f0 + fl;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int band = lane + 32 * h;
            const int lo = S.fb_lo[band], cnt = S.fb_cnt[band];
            const double *w = S.fbw + S.fb_off[band];
            double acc = 0.0;
            for (int b = 0; b < cnt; ++b) { const int k = lo + b; acc += pw[k + (k >> 5)] * w[b]; }
            raw[f * VBANDS + band] = log(fmax(1.0, acc));
        }
        __syncwarp();
    }
}

// (32 CTAs of 64 threads per SM, as before the record table: the lookup fits the 32 registers without spills)
__global__ void __launch_bounds__(VBANDS, 32)
vbx_cmvn_kernel(const VbxRec *__restrict__ recs, int n_rec, const double *__restrict__ raw_all, float *__restrict__ fea_all)
{
    const int band = threadIdx.x;
    const VbxRec &rec = find_rec<&VbxRec::chunk_off>(recs, n_rec, blockIdx.x);
    const int64_t M = rec.M;                            // the window never leaves this recording's rows
    const double *raw = raw_all + rec.raw_off * VBANDS;
    float *fea = fea_all + rec.fea_off * VBANDS;
    const int64_t t0 = ((int64_t)blockIdx.x - rec.chunk_off) * CMVN_CHUNK;
    const int64_t t1 = min(t0 + CMVN_CHUNK, M);
    const int64_t wl = min(M, (int64_t)CMVN_WIN);
    auto wstart = [&](int64_t t) { return max(min(t - CMVN_LC, M - wl), (int64_t)0); };
    int64_t ws = wstart(t0);
    double sum = 0.0;
    for (int64_t r = ws; r < ws + wl; ++r) sum += raw[r * VBANDS + band];
    for (int64_t t = t0; t < t1; ++t) {
        const int64_t nws = wstart(t);
        if (nws != ws) {                                // the window slides by exactly one row
            sum += raw[(nws + wl - 1) * VBANDS + band] - raw[ws * VBANDS + band];
            ws = nws;
        }
        fea[t * VBANDS + band] = (float)(raw[t * VBANDS + band] - sum / (double)wl);
    }
}

}  // namespace

static VbxTables *g_vbx_tables[64] = {nullptr};        // per device

extern "C" int64_t iss_vbx_num_frames(int64_t n_samples)
{
    if (n_samples < VPADR) return 0;                    // mirror padding needs >= 200 samples
    return (n_samples + VPADL + VPADR - ISS_WIN) / ISS_HOP + 1;
}

extern "C" int iss_vbx_upload_tables(iss_ctx *ctx, const double *h_fbank, const double *h_window)
{
    ISS_REQUIRE(ctx && h_fbank && h_window, ISS_ERR_INVALID, "iss_vbx_upload_tables: NULL argument");
    ISS_REQUIRE(ctx->device < 64, ISS_ERR_INVALID, "device index");
    ISS_CUDA_OK(cudaSetDevice(ctx->device));
    VbxTables *t = new VbxTables();
    memset(t, 0, sizeof(*t));
    int nnz = 0;
    for (int m = 0; m < VBANDS; ++m) {                  // h_fbank is [257][64] (features_vbx.py:31-59)
        int lo = -1, hi = -1;
        for (int k = 0; k < ISS_NBIN; ++k)
            if (h_fbank[k * VBANDS + m] != 0.0) { if (lo < 0) lo = k; hi = k; }
        t->lo[m] = lo < 0 ? 0 : lo;
        t->cnt[m] = lo < 0 ? 0 : hi - lo + 1;
        t->off[m] = nnz;
        if (nnz + t->cnt[m] > VMAXNNZ) { delete t; iss_set_error("iss_vbx_upload_tables: filterbank too wide"); return ISS_ERR_INVALID; }
        for (int b = 0; b < t->cnt[m]; ++b) t->w[nnz++] = h_fbank[(lo + b) * VBANDS + m];
    }
    t->nnz = nnz;
    const double PI = 3.14159265358979323846;
    for (int i = 0; i < ISS_WIN; ++i) t->win[i] = h_window[i];
    for (int m = 0; m < 256; ++m) { t->tw256[2 * m] = cos(2.0 * PI * m / 256.0); t->tw256[2 * m + 1] = -sin(2.0 * PI * m / 256.0); }
    for (int k = 0; k <= 256; ++k) { t->tw512[2 * k] = cos(2.0 * PI * k / 512.0); t->tw512[2 * k + 1] = -sin(2.0 * PI * k / 512.0); }
    VbxTables *&d = g_vbx_tables[ctx->device];
    if (!d) {
        cudaError_t e = cudaMalloc(&d, sizeof(VbxTables));
        if (e != cudaSuccess) { delete t; iss_set_error("cudaMalloc vbx tables: %s", cudaGetErrorString(e)); return ISS_ERR_NOMEM; }
    }
    cudaError_t e = cudaMemcpy(d, t, sizeof(VbxTables), cudaMemcpyHostToDevice);
    delete t;
    if (e != cudaSuccess) { iss_set_error("cudaMemcpy vbx tables: %s", cudaGetErrorString(e)); return ISS_ERR_CUDA; }
    return ISS_OK;
}

extern "C" int64_t iss_vbx_work_bytes(int64_t n_samples)
{
    return iss_vbx_num_frames(n_samples) * VBANDS * (int64_t)sizeof(double) + 256;
}

extern "C" int iss_vbx_features_multi(iss_ctx *ctx, int n_rec, const void *const *h_pcm, const int64_t *h_n_samples,
                                      int pcm_format, const double *d_dither, float *d_fea, const int64_t *h_fea_off,
                                      void *d_work, void *stream)
{
    ISS_REQUIRE(ctx, ISS_ERR_INVALID, "iss_vbx_features: ctx is NULL");
    ISS_REQUIRE(ctx->device < 64 && g_vbx_tables[ctx->device], ISS_ERR_STATE, "iss_vbx_features: call iss_vbx_upload_tables first");
    ISS_REQUIRE(pcm_format == ISS_PCM_F32 || pcm_format == ISS_PCM_S16, ISS_ERR_INVALID, "bad pcm_format %d", pcm_format);
    ISS_REQUIRE(n_rec >= 1 && h_pcm && h_n_samples && h_fea_off, ISS_ERR_INVALID, "iss_vbx_features_multi: bad argument");
    std::vector<VbxRec> recs(n_rec + 1);
    int64_t rows = 0, ntiles = 0, nchunks = 0;
    for (int i = 0; i < n_rec; ++i) {
        VbxRec &r = recs[i];
        r.pcm = h_pcm[i];
        r.n = h_n_samples[i];
        r.M = iss_vbx_num_frames(r.n);
        r.raw_off = rows; r.fea_off = h_fea_off[i]; r.tile_off = ntiles; r.chunk_off = nchunks;
        ISS_REQUIRE(r.M == 0 || r.pcm, ISS_ERR_INVALID, "iss_vbx_features: NULL buffer (recording %d)", i);
        ISS_REQUIRE(r.fea_off >= 0, ISS_ERR_INVALID, "iss_vbx_features_multi: negative offset (recording %d)", i);
        rows += r.M;
        ntiles += (r.M + VFR - 1) / VFR;
        nchunks += (r.M + CMVN_CHUNK - 1) / CMVN_CHUNK;
    }
    recs[n_rec] = VbxRec{nullptr, 0, 0, rows, 0, ntiles, nchunks};
    if (rows == 0) return ISS_OK;
    ISS_REQUIRE(d_fea && d_work, ISS_ERR_INVALID, "iss_vbx_features: NULL buffer");
    ISS_REQUIRE(ntiles < (1ll << 31), ISS_ERR_INVALID, "iss_vbx_features: signal too long for one call");
    ISS_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = iss_stream(stream);
    if (n_rec + 1 > ctx->vbx_recs_cap) {
        if (ctx->d_vbx_recs) ISS_CUDA_OK(cudaFree(ctx->d_vbx_recs));
        ctx->d_vbx_recs = nullptr; ctx->vbx_recs_cap = 0;
        const int64_t cap = n_rec + 1 + n_rec / 2 + 64;
        cudaError_t e = cudaMalloc(&ctx->d_vbx_recs, (size_t)cap * sizeof(VbxRec));
        if (e != cudaSuccess) { iss_set_error("cudaMalloc recording table: %s", cudaGetErrorString(e)); return ISS_ERR_NOMEM; }
        ctx->vbx_recs_cap = cap;
    }
    const VbxRec *d_recs = reinterpret_cast<const VbxRec *>(ctx->d_vbx_recs);
    ISS_CUDA_OK(cudaMemcpyAsync(ctx->d_vbx_recs, recs.data(), sizeof(VbxRec) * (n_rec + 1), cudaMemcpyHostToDevice, st));
    double *raw = reinterpret_cast<double *>(d_work);
    const size_t smem = sizeof(VSmem);
    if (pcm_format == ISS_PCM_S16) {
        ISS_CUDA_OK(cudaFuncSetAttribute(vbx_fbank_kernel<ISS_PCM_S16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        vbx_fbank_kernel<ISS_PCM_S16><<<(unsigned)ntiles, VNTHREAD, smem, st>>>(d_recs, n_rec, d_dither, g_vbx_tables[ctx->device], raw);
    } else {
        ISS_CUDA_OK(cudaFuncSetAttribute(vbx_fbank_kernel<ISS_PCM_F32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        vbx_fbank_kernel<ISS_PCM_F32><<<(unsigned)ntiles, VNTHREAD, smem, st>>>(d_recs, n_rec, d_dither, g_vbx_tables[ctx->device], raw);
    }
    ISS_CUDA_OK(cudaGetLastError());
    vbx_cmvn_kernel<<<(unsigned)nchunks, VBANDS, 0, st>>>(d_recs, n_rec, raw, d_fea);
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch(2);
    return ISS_OK;
}

extern "C" int iss_vbx_features(iss_ctx *ctx, const void *d_pcm, int pcm_format, int64_t n_samples,
                                const double *d_dither, float *d_fea, void *d_work, void *stream)
{
    const int64_t zero = 0;
    return iss_vbx_features_multi(ctx, 1, &d_pcm, &n_samples, pcm_format, d_dither, d_fea, &zero, d_work, stream);
}
