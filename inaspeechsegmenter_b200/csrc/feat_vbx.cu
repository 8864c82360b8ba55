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
// MT19937 sequence (np.random.seed(3)), so it is an input stream: a device-resident
// prefix for whole recordings, or, for live streams, drawn call by call from one
// MT19937 state per stream (dither_mt19937_kernel).
//
// Kernel A: tile of FR frames per CTA, padded/dithered samples staged once in shared
// memory as doubles, one frame per warp iteration, FFT from fft256.cuh, sparse 64-band
// filterbank, raw log-fbank written as float64 [M][64] to scratch.
// Kernel B: sliding 300-frame mean (Kaldi edge handling: the window shifts, it does
// not shrink), one thread per band, 128-frame chunks: direct sum for the first frame
// of the chunk, then add/subtract one row per step.
// Both kernels take a table of windowed records (a whole recording is one window): a CTA
// finds its record by binary search over the tile / chunk offsets, and every index inside
// it (padding, dither, tile, CMVN window) is local to that record's stream.
#include <math.h>
#include <string.h>
#include <algorithm>
#include <utility>
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

// One window of one stream in an fbank call: the record holds samples [s_base, s_known) (pcm and dither, both indexed
// from s_base) and computes raw rows [r_first, r_first + rows) into raw rows raw_off .. of the scratch.  Its tiles are
// [tile_off, next record's tile_off); tile t starts at row r_first + VFR * (t - tile_off).  A recording read whole is the
// window s_base = r_first = 0, s_known = n, rows = M: every row is a function of its own 400 padded samples only, so
// where a tile starts does not change it.  The right mirror reads around s_known, which the host allows only once the
// stream has ended.
struct VbxFbRec {
    const void *pcm;
    const double *dither;           // NULL: no dither
    int64_t s_base, s_known;
    int64_t r_first, rows;
    int64_t raw_off;
    int64_t tile_off;               // first fbank tile (global block index); entry n_rec holds the total
};

// One window of CMVN rows: raw rows [r_base, r_known) sit at scratch rows raw_off .., feature rows [t_first,
// t_first + rows) go to output rows fea_off ...  M = r_known: the rows a record may ask for (checked on the host) are
// those whose window no longer depends on later rows, or all of them once the stream has ended.  Each CTA replays one
// 128-row chunk of the grid of the whole recording from its start (direct sum, then add / subtract), so a row comes out
// of the same adds in the same order whichever window computes it.
struct VbxCmRec {
    int64_t r_base, r_known;
    int64_t t_first, rows;
    int64_t raw_off, fea_off;
    int64_t chunk_off;              // first CMVN chunk (global block index); entry n_rec holds the total
};

// recs[lo].off <= b < recs[hi].off (records without rows own no block)
template <typename R>
__device__ __forceinline__ const R &find_rec(const R *__restrict__ recs, int n_rec, int64_t b, int64_t R::*off)
{
    int lo = 0, hi = n_rec;
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (recs[mid].*off <= b) lo = mid; else hi = mid; }
    return recs[lo];
}

template <int PCM>
__global__ void __launch_bounds__(VNTHREAD, 2)
vbx_fbank_kernel(const VbxFbRec *__restrict__ recs, int n_rec, const VbxTables *__restrict__ tabs, double *__restrict__ raw_all)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    VSmem &S = *reinterpret_cast<VSmem *>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const VbxFbRec &rec = find_rec(recs, n_rec, blockIdx.x, &VbxFbRec::tile_off);
    const void *pcm = rec.pcm;
    const double *dither = rec.dither;
    const int64_t n = rec.s_known, s_base = rec.s_base;
    const int64_t tf = ((int64_t)blockIdx.x - rec.tile_off) * VFR;
    double *raw = raw_all + (rec.raw_off + tf) * VBANDS;
    const int64_t f0 = rec.r_first + tf;
    const int nfr = (int)min((int64_t)VFR, rec.rows - tf);
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
        src -= s_base;
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
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int band = lane + 32 * h;
            const int lo = S.fb_lo[band], cnt = S.fb_cnt[band];
            const double *w = S.fbw + S.fb_off[band];
            double acc = 0.0;
            for (int b = 0; b < cnt; ++b) { const int k = lo + b; acc += pw[k + (k >> 5)] * w[b]; }
            raw[fl * VBANDS + band] = log(fmax(1.0, acc));
        }
        __syncwarp();
    }
}

// (32 CTAs of 64 threads per SM, as before the record table: the lookup fits the 32 registers without spills)
__global__ void __launch_bounds__(VBANDS, 32)
vbx_cmvn_kernel(const VbxCmRec *__restrict__ recs, int n_rec, const double *__restrict__ raw_all, float *__restrict__ fea_all)
{
    const int band = threadIdx.x;
    const VbxCmRec &rec = find_rec(recs, n_rec, blockIdx.x, &VbxCmRec::chunk_off);
    const int64_t M = rec.r_known;                      // the window never leaves the record's known rows
    const double *raw = raw_all + (rec.raw_off - rec.r_base) * VBANDS;      // indexed by the stream's row number
    float *fea = fea_all + (rec.fea_off - rec.t_first) * VBANDS;
    const int64_t t0 = (rec.t_first / CMVN_CHUNK + ((int64_t)blockIdx.x - rec.chunk_off)) * CMVN_CHUNK;
    const int64_t ta = max(t0, rec.t_first);
    const int64_t t1 = min(t0 + CMVN_CHUNK, rec.t_first + rec.rows);
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
        if (t >= ta) fea[t * VBANDS + band] = (float)(raw[t * VBANDS + band] - sum / (double)wl);
    }
}

// One MT19937 state per stream slot: state[slot * 625 ..] holds the 624 key words, then the position of the next word
// (624: twist first), as numpy's RandomState.get_state() gives them.  A record draws the slot's next `n` doubles the way
// the legacy RandomState.rand does (two tempered words a, b -> ((a >> 5) 2^26 + (b >> 6)) / 2^53, every step exact) and
// writes the dither 8 (2u - 1) of each to out[out_off ..].  The position stays even (whole doubles are drawn from a
// state that starts at 624), so a double never straddles a twist; a position that is odd or past 624 is taken as 624.
struct DitherRec {
    int64_t slot, n, out_off;
};

constexpr int MT_N = 624, MT_M = 397, MT_THREADS = 256;

__global__ void __launch_bounds__(MT_THREADS)
dither_mt19937_kernel(const DitherRec *__restrict__ recs, uint32_t *__restrict__ state, double *__restrict__ out)
{
    __shared__ uint32_t mt[MT_N];
    const DitherRec rec = recs[blockIdx.x];
    uint32_t *g = state + rec.slot * (MT_N + 1);
    const int tid = threadIdx.x;
    for (int i = tid; i < MT_N; i += MT_THREADS) mt[i] = g[i];
    // a position the table cannot hold (odd, or past 624) is read as 624, the twist; it never stalls the draw loop
    const uint32_t gpos = g[MT_N];
    int pos = (gpos <= (uint32_t)MT_N && !(gpos & 1u)) ? (int)gpos : MT_N;
    __syncthreads();
    double *o = out + rec.out_off;
    for (int64_t k = 0; k < rec.n;) {
        if (pos >= MT_N) {
            // the twist in its three dependent phases: [0, 227) reads old words only, [227, 454) reads words of the
            // first phase (i + 397 - 624), [454, 624) words of the second (and word 0 for i = 623)
            for (int lo = 0; lo < MT_N; lo += MT_N - MT_M) {
                const int hi = min(lo + MT_N - MT_M, MT_N), i = lo + tid;
                uint32_t v = 0;
                if (i < hi) {
                    const uint32_t y = (mt[i] & 0x80000000u) | (mt[i + 1 < MT_N ? i + 1 : 0] & 0x7fffffffu);
                    v = mt[i + MT_M < MT_N ? i + MT_M : i + MT_M - MT_N] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
                }
                __syncthreads();
                if (i < hi) mt[i] = v;
                __syncthreads();
            }
            pos = 0;
        }
        const int64_t m = min((int64_t)(MT_N - pos) / 2, rec.n - k);
        for (int j = tid; j < m; j += MT_THREADS) {
            uint32_t w[2] = {mt[pos + 2 * j], mt[pos + 2 * j + 1]};
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                uint32_t y = w[h];
                y ^= y >> 11;
                y ^= (y << 7) & 0x9d2c5680u;
                y ^= (y << 15) & 0xefc60000u;
                y ^= y >> 18;
                w[h] = y;
            }
            const double u = ((double)(w[0] >> 5) * 67108864.0 + (double)(w[1] >> 6)) / 9007199254740992.0;
            o[k + j] = 8.0 * (u * 2.0 - 1.0);
        }
        pos += 2 * (int)m;
        k += m;
        __syncthreads();
    }
    for (int i = tid; i < MT_N; i += MT_THREADS) g[i] = mt[i];
    if (tid == 0) g[MT_N] = (uint32_t)pos;
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

// Copies a host record table to the context's device table (grown as needed), in stream order.
static int upload_recs(iss_ctx *ctx, const void *h, size_t bytes, cudaStream_t st, const void **d)
{
    if ((int64_t)bytes > ctx->vbx_recs_cap) {
        if (ctx->d_vbx_recs) ISS_CUDA_OK(cudaFree(ctx->d_vbx_recs));
        ctx->d_vbx_recs = nullptr; ctx->vbx_recs_cap = 0;
        const int64_t cap = (int64_t)bytes + (int64_t)bytes / 2 + 4096;
        cudaError_t e = cudaMalloc(&ctx->d_vbx_recs, (size_t)cap);
        if (e != cudaSuccess) { iss_set_error("cudaMalloc record table: %s", cudaGetErrorString(e)); return ISS_ERR_NOMEM; }
        ctx->vbx_recs_cap = cap;
    }
    ISS_CUDA_OK(cudaMemcpyAsync(ctx->d_vbx_recs, h, bytes, cudaMemcpyHostToDevice, st));
    *d = ctx->d_vbx_recs;
    return ISS_OK;
}

static int check_ctx(iss_ctx *ctx, const char *fn)
{
    ISS_REQUIRE(ctx, ISS_ERR_INVALID, "%s: ctx is NULL", fn);
    ISS_REQUIRE(ctx->device < 64 && g_vbx_tables[ctx->device], ISS_ERR_STATE, "%s: call iss_vbx_upload_tables first", fn);
    return ISS_OK;
}

// Both kernels over finished record tables (entry n_rec of each holds the totals); the fbank table is recs[0 ..
// n_fb], the CMVN table follows it.  Either table may be empty (n = 0).
static int launch(iss_ctx *ctx, int pcm_format, const std::vector<VbxFbRec> &fb, const std::vector<VbxCmRec> &cm,
                  double *raw, float *fea, void *stream)
{
    const int n_fb = (int)fb.size() - 1, n_cm = (int)cm.size() - 1;
    const int64_t ntiles = n_fb > 0 ? fb[n_fb].tile_off : 0, nchunks = n_cm > 0 ? cm[n_cm].chunk_off : 0;
    if (ntiles == 0 && nchunks == 0) return ISS_OK;
    ISS_REQUIRE(ntiles < (1ll << 31) && nchunks < (1ll << 31), ISS_ERR_INVALID, "iss_vbx: too many rows for one call");
    ISS_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = iss_stream(stream);
    const size_t fb_bytes = ntiles ? fb.size() * sizeof(VbxFbRec) : 0;
    std::vector<unsigned char> h(fb_bytes + (nchunks ? cm.size() * sizeof(VbxCmRec) : 0));
    if (ntiles) memcpy(h.data(), fb.data(), fb_bytes);
    if (nchunks) memcpy(h.data() + fb_bytes, cm.data(), cm.size() * sizeof(VbxCmRec));
    const void *d = nullptr;
    int rc = upload_recs(ctx, h.data(), h.size(), st, &d);
    if (rc != ISS_OK) return rc;
    int launches = 0;
    if (ntiles) {
        const VbxFbRec *d_fb = reinterpret_cast<const VbxFbRec *>(d);
        const size_t smem = sizeof(VSmem);
        if (pcm_format == ISS_PCM_S16) {
            ISS_CUDA_OK(cudaFuncSetAttribute(vbx_fbank_kernel<ISS_PCM_S16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            vbx_fbank_kernel<ISS_PCM_S16><<<(unsigned)ntiles, VNTHREAD, smem, st>>>(d_fb, n_fb, g_vbx_tables[ctx->device], raw);
        } else {
            ISS_CUDA_OK(cudaFuncSetAttribute(vbx_fbank_kernel<ISS_PCM_F32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            vbx_fbank_kernel<ISS_PCM_F32><<<(unsigned)ntiles, VNTHREAD, smem, st>>>(d_fb, n_fb, g_vbx_tables[ctx->device], raw);
        }
        ISS_CUDA_OK(cudaGetLastError());
        ++launches;
    }
    if (nchunks) {
        const VbxCmRec *d_cm = reinterpret_cast<const VbxCmRec *>(reinterpret_cast<const unsigned char *>(d) + fb_bytes);
        vbx_cmvn_kernel<<<(unsigned)nchunks, VBANDS, 0, st>>>(d_cm, n_cm, raw, fea);
        ISS_CUDA_OK(cudaGetLastError());
        ++launches;
    }
    iss_count_launch(launches);
    return ISS_OK;
}

static int64_t cmvn_chunks(int64_t t_first, int64_t rows)
{
    return rows > 0 ? (t_first + rows - 1) / CMVN_CHUNK - t_first / CMVN_CHUNK + 1 : 0;
}

extern "C" int iss_vbx_features_multi(iss_ctx *ctx, int n_rec, const void *const *h_pcm, const int64_t *h_n_samples,
                                      int pcm_format, const double *d_dither, float *d_fea, const int64_t *h_fea_off,
                                      void *d_work, void *stream)
{
    int rc = check_ctx(ctx, "iss_vbx_features");
    if (rc != ISS_OK) return rc;
    ISS_REQUIRE(pcm_format == ISS_PCM_F32 || pcm_format == ISS_PCM_S16, ISS_ERR_INVALID, "bad pcm_format %d", pcm_format);
    ISS_REQUIRE(n_rec >= 1 && h_pcm && h_n_samples && h_fea_off, ISS_ERR_INVALID, "iss_vbx_features_multi: bad argument");
    // every recording is the window s_base = r_first = r_base = t_first = 0 of a stream that has ended
    std::vector<VbxFbRec> fb(n_rec + 1);
    std::vector<VbxCmRec> cm(n_rec + 1);
    int64_t rows = 0, ntiles = 0, nchunks = 0;
    for (int i = 0; i < n_rec; ++i) {
        const int64_t n = h_n_samples[i], M = iss_vbx_num_frames(n);
        ISS_REQUIRE(M == 0 || h_pcm[i], ISS_ERR_INVALID, "iss_vbx_features: NULL buffer (recording %d)", i);
        ISS_REQUIRE(h_fea_off[i] >= 0, ISS_ERR_INVALID, "iss_vbx_features_multi: negative offset (recording %d)", i);
        fb[i] = VbxFbRec{h_pcm[i], d_dither, 0, n, 0, M, rows, ntiles};
        cm[i] = VbxCmRec{0, M, 0, M, rows, h_fea_off[i], nchunks};
        rows += M;
        ntiles += (M + VFR - 1) / VFR;
        nchunks += cmvn_chunks(0, M);
    }
    fb[n_rec] = VbxFbRec{nullptr, nullptr, 0, 0, 0, 0, rows, ntiles};
    cm[n_rec] = VbxCmRec{0, 0, 0, 0, rows, 0, nchunks};
    if (rows == 0) return ISS_OK;
    ISS_REQUIRE(d_fea && d_work, ISS_ERR_INVALID, "iss_vbx_features: NULL buffer");
    return launch(ctx, pcm_format, fb, cm, reinterpret_cast<double *>(d_work), d_fea, stream);
}

extern "C" int iss_vbx_features(iss_ctx *ctx, const void *d_pcm, int pcm_format, int64_t n_samples,
                                const double *d_dither, float *d_fea, void *d_work, void *stream)
{
    const int64_t zero = 0;
    return iss_vbx_features_multi(ctx, 1, &d_pcm, &n_samples, pcm_format, d_dither, d_fea, &zero, d_work, stream);
}

extern "C" int iss_vbx_fbank_window_multi(iss_ctx *ctx, int n_rec, const void *const *h_pcm,
                                          const double *const *h_dither, const int64_t *h_win, int pcm_format,
                                          double *d_raw, void *stream)
{
    const char *fn = "iss_vbx_fbank_window_multi";
    int rc = check_ctx(ctx, fn);
    if (rc != ISS_OK) return rc;
    ISS_REQUIRE(pcm_format == ISS_PCM_F32 || pcm_format == ISS_PCM_S16, ISS_ERR_INVALID, "bad pcm_format %d", pcm_format);
    ISS_REQUIRE(n_rec >= 1 && h_pcm && h_dither && h_win, ISS_ERR_INVALID, "%s: bad argument", fn);
    std::vector<VbxFbRec> fb(n_rec + 1);
    int64_t ntiles = 0;
    for (int i = 0; i < n_rec; ++i) {
        const int64_t *w = h_win + (size_t)i * 6;
        const int64_t s_base = w[0], s_known = w[1], r_first = w[2], rows = w[3], raw_off = w[4], flags = w[5];
        ISS_REQUIRE(s_base >= 0 && s_base <= s_known && s_known < ((int64_t)1 << 40) && r_first >= 0 && rows >= 0 &&
                    raw_off >= 0 && (flags & ~(int64_t)ISS_VBX_END) == 0, ISS_ERR_INVALID, "%s: record %d: bad field", fn, i);
        if (rows > 0) {
            const int64_t last = r_first + rows - 1;
            ISS_REQUIRE(h_pcm[i], ISS_ERR_INVALID, "%s: record %d: NULL buffer", fn, i);
            // row r reads samples max(0, 160 r - 120) .. 160 r + 279, or mirrored ones at or after the first of these
            const int64_t first = r_first * ISS_HOP - VPADL > 0 ? r_first * ISS_HOP - VPADL : 0;
            ISS_REQUIRE(first >= s_base, ISS_ERR_INVALID, "%s: record %d: row %lld reads sample %lld, before the window's "
                        "first sample %lld", fn, i, (long long)r_first, (long long)first, (long long)s_base);
            if (flags & ISS_VBX_END)
                ISS_REQUIRE(last < iss_vbx_num_frames(s_known), ISS_ERR_INVALID, "%s: record %d: row %lld past the %lld "
                            "rows of %lld samples", fn, i, (long long)last, (long long)iss_vbx_num_frames(s_known),
                            (long long)s_known);
            else
                ISS_REQUIRE(last * ISS_HOP + ISS_WIN - VPADL <= s_known, ISS_ERR_INVALID, "%s: record %d: row %lld reads "
                            "sample %lld of %lld known samples, and the stream has not ended", fn, i, (long long)last,
                            (long long)(last * ISS_HOP + ISS_WIN - VPADL - 1), (long long)s_known);
        }
        fb[i] = VbxFbRec{h_pcm[i], h_dither[i], s_base, s_known, r_first, rows, raw_off, ntiles};
        ntiles += (rows + VFR - 1) / VFR;
    }
    fb[n_rec] = VbxFbRec{nullptr, nullptr, 0, 0, 0, 0, 0, ntiles};
    ISS_REQUIRE(ntiles == 0 || d_raw, ISS_ERR_INVALID, "%s: NULL output", fn);
    return launch(ctx, pcm_format, fb, std::vector<VbxCmRec>(1), d_raw, nullptr, stream);
}

extern "C" int iss_vbx_cmvn_window_multi(iss_ctx *ctx, int n_rec, const int64_t *h_win, const double *d_raw,
                                         float *d_fea, void *stream)
{
    const char *fn = "iss_vbx_cmvn_window_multi";
    int rc = check_ctx(ctx, fn);
    if (rc != ISS_OK) return rc;
    ISS_REQUIRE(n_rec >= 1 && h_win, ISS_ERR_INVALID, "%s: bad argument", fn);
    std::vector<VbxCmRec> cm(n_rec + 1);
    int64_t nchunks = 0;
    for (int i = 0; i < n_rec; ++i) {
        const int64_t *w = h_win + (size_t)i * 7;
        const int64_t r_base = w[0], r_known = w[1], t_first = w[2], rows = w[3], raw_off = w[4], fea_off = w[5], flags = w[6];
        ISS_REQUIRE(r_base >= 0 && r_base <= r_known && r_known < ((int64_t)1 << 40) && t_first >= 0 && rows >= 0 &&
                    raw_off >= 0 && fea_off >= 0 && (flags & ~(int64_t)ISS_VBX_END) == 0, ISS_ERR_INVALID,
                    "%s: record %d: bad field", fn, i);
        if (rows > 0) {
            const int64_t last = t_first + rows - 1, wl = r_known < CMVN_WIN ? r_known : CMVN_WIN;
            ISS_REQUIRE(last < r_known, ISS_ERR_INVALID, "%s: record %d: row %lld of %lld rows", fn, i, (long long)last,
                        (long long)r_known);
            // a row's window no longer moves once 150 rows follow it and 300 exist; before the end, only such rows
            ISS_REQUIRE((flags & ISS_VBX_END) || (r_known >= CMVN_WIN && last + CMVN_LC <= r_known), ISS_ERR_INVALID,
                        "%s: record %d: row %lld is not final with %lld known rows, and the stream has not ended", fn, i,
                        (long long)last, (long long)r_known);
            // the chunk of t_first starts with a direct sum from its own window start
            const int64_t c0 = t_first / CMVN_CHUNK * CMVN_CHUNK;
            int64_t ws = c0 - CMVN_LC < r_known - wl ? c0 - CMVN_LC : r_known - wl;
            ws = ws > 0 ? ws : 0;
            ISS_REQUIRE(ws >= r_base, ISS_ERR_INVALID, "%s: record %d: the chunk of row %lld reads row %lld, before the "
                        "window's first row %lld", fn, i, (long long)t_first, (long long)ws, (long long)r_base);
        }
        cm[i] = VbxCmRec{r_base, r_known, t_first, rows, raw_off, fea_off, nchunks};
        nchunks += cmvn_chunks(t_first, rows);
    }
    cm[n_rec] = VbxCmRec{0, 0, 0, 0, 0, 0, nchunks};
    ISS_REQUIRE(nchunks == 0 || (d_raw && d_fea), ISS_ERR_INVALID, "%s: NULL buffer", fn);
    return launch(ctx, ISS_PCM_F32, std::vector<VbxFbRec>(1), cm, const_cast<double *>(d_raw), d_fea, stream);
}

extern "C" int iss_dither_mt19937_multi(iss_ctx *ctx, int n_rec, const int64_t *h_rec, uint32_t *d_state,
                                        int64_t n_slots, double *d_out, void *stream)
{
    const char *fn = "iss_dither_mt19937_multi";
    ISS_REQUIRE(ctx, ISS_ERR_INVALID, "%s: ctx is NULL", fn);
    ISS_REQUIRE(n_rec >= 1 && h_rec && n_slots >= 0, ISS_ERR_INVALID, "%s: bad argument", fn);
    ISS_REQUIRE(n_slots < ((int64_t)1 << 31), ISS_ERR_INVALID, "%s: %lld slots", fn, (long long)n_slots);
    std::vector<DitherRec> recs;
    std::vector<std::pair<int64_t, int>> slots;         // (slot, record): a slot drawn twice is found by sorting
    for (int i = 0; i < n_rec; ++i) {
        const int64_t slot = h_rec[3 * i], n = h_rec[3 * i + 1], off = h_rec[3 * i + 2];
        ISS_REQUIRE(slot >= 0 && slot < n_slots && n >= 0 && n < ((int64_t)1 << 40) && off >= 0, ISS_ERR_INVALID,
                    "%s: record %d: bad field", fn, i);
        slots.emplace_back(slot, i);
        if (n) recs.push_back(DitherRec{slot, n, off});
    }
    std::sort(slots.begin(), slots.end());
    for (size_t j = 1; j < slots.size(); ++j)
        ISS_REQUIRE(slots[j].first != slots[j - 1].first, ISS_ERR_INVALID, "%s: record %d: slot %lld drawn twice in one "
                    "call", fn, slots[j].second, (long long)slots[j].first);
    if (recs.empty()) return ISS_OK;
    ISS_REQUIRE(d_state && d_out, ISS_ERR_INVALID, "%s: NULL buffer", fn);
    ISS_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = iss_stream(stream);
    const void *d = nullptr;
    int rc = upload_recs(ctx, recs.data(), recs.size() * sizeof(DitherRec), st, &d);
    if (rc != ISS_OK) return rc;
    dither_mt19937_kernel<<<(unsigned)recs.size(), MT_THREADS, 0, st>>>(reinterpret_cast<const DitherRec *>(d), d_state, d_out);
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch();
    return ISS_OK;
}
