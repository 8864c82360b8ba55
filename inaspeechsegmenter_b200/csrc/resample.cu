// resample.cu -- downmix + polyphase FIR resampling of PCM (int16, float32, and the WAV encodings unsigned 8-bit,
// packed 24-bit, int32 and float64) to 16 kHz mono int16.
//
// Definition (DESIGN.md "Resampling"): a recording of n frames, C channels at integer rate R is
//   x[m]  = mean over the C channels of frame m in float64 (int16 s as s / 32768, float32 as is; pcm_value below),
//   y[k]  = scipy.signal.resample_poly(x, up, down)[k],  up = 16000 / g, down = R / g, g = gcd(16000, R),
//         = sum_m x[m] h[k * down + H - m * up]  with h the 2H + 1 taps (H = 10 max(up, down)) of scipy's
//           default design times up, and x = 0 outside [0, n),
//   out[k] = clip(rint(y[k] * 32768), -32768, 32767) as int16,   k < ceil(n * up / down).
// The host designs h (resample.py); iss_resample_upload_taps arranges it by phase: output k, with
// k * down = a * up + q, needs the taps of phase q against the frames a + s_q .. a + s_q + n_q - 1, ascending.
//
// Layout: one CTA owns a tile of consecutive outputs of one record (tiles start at the record's first output k_first).
// It stages the raw samples of the tile's input span in shared memory with 16-byte loads (scalar loads when the
// record's base pointer is not 16-byte aligned, byte loads when it is not even aligned to its samples, as a WAV's
// stored bytes may lie at any address; packed 24-bit samples are staged as bytes and sign-extended in the downmix),
// downmixes them there into float64, then each thread evaluates
// its outputs as float64 FMA chains in ascending frame order.  No atomics, and no value depends on the tiling.
//
// Windows (live streams): a record's buffer holds frames [f_base, n_known) of its stream, and it computes outputs
// [k_first, k_first + n_out).  Frames at or past n_known read as zero, as do frames before 0.  A whole recording is
// the window f_base = 0, k_first = 0, n_out = ceil(n * up / down); iss_resample_window_multi checks on the host that
// no output of a window reads a frame in [0, f_base), and that only a stream's final outputs read past n_known.
#include <math.h>
#include <string.h>

#include <map>
#include <vector>

#include "iss_common.cuh"

namespace {

constexpr int RS_THREADS = 256;
constexpr int RS_TARGET = 16000;
constexpr int RS_MIN_RATE = 8000, RS_MAX_RATE = 192000, RS_MAX_CHANNELS = 8;
constexpr int RS_SMEM_BUDGET = 96 * 1024;            // two CTAs per SM
constexpr int RS_MAX_TILE = 1024, RS_MIN_TILE = 32;

struct Phase {
    int off;                 // first tap of the phase in the packed tap array
    int n;                   // taps
    int s;                   // first input frame relative to a = floor(k * down / up)
    int pad;
};

// One record (a recording, or a window of a stream) of a resampling call.  Its tiles are [tile_off, next record's
// tile_off).
struct RsRec {
    const void *pcm;                // frame f_base of the stream
    int64_t f_base;
    int64_t n_known;                // frames >= n_known are zero
    int64_t k_first;
    int64_t n_out;
    int64_t out_off;                // int16 element of output k_first
    int64_t tile_off;               // first tile (global block index); entry n_rec holds the total
    int align;                      // pcm is 16-byte aligned (2), aligned to its Unit (1), or neither (0)
};

// A stored sample is UNITS consecutive Units (what the staging loads: bytes for packed 24-bit) in record order.
template <int PCM> struct PcmIn;
template <> struct PcmIn<ISS_PCM_F32> { using Unit = float;   static constexpr int UNITS = 1; };
template <> struct PcmIn<ISS_PCM_S16> { using Unit = int16_t; static constexpr int UNITS = 1; };
template <> struct PcmIn<ISS_PCM_U8>  { using Unit = uint8_t; static constexpr int UNITS = 1; };
template <> struct PcmIn<ISS_PCM_S24> { using Unit = uint8_t; static constexpr int UNITS = 3; };
template <> struct PcmIn<ISS_PCM_S32> { using Unit = int32_t; static constexpr int UNITS = 1; };
template <> struct PcmIn<ISS_PCM_F64> { using Unit = double;  static constexpr int UNITS = 1; };

// Step 1 of the definition: the stored sample at p as float64.  Every scale is a power of two, so each value is exact.
template <int PCM>
__device__ __forceinline__ double pcm_value(const typename PcmIn<PCM>::Unit *p)
{
    if constexpr (PCM == ISS_PCM_S16) return (double)p[0] * (1.0 / 32768.0);
    else if constexpr (PCM == ISS_PCM_U8) return (double)((int)p[0] - 128) * (1.0 / 128.0);
    else if constexpr (PCM == ISS_PCM_S24)        // little-endian; the shift pair sign-extends bit 23
        return (double)((int)(((uint32_t)p[0] << 8) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 24)) >> 8) *
               (1.0 / 8388608.0);
    else if constexpr (PCM == ISS_PCM_S32) return (double)p[0] * (1.0 / 2147483648.0);
    else return (double)p[0];                     // float32, float64
}

template <int PCM>
__global__ void __launch_bounds__(RS_THREADS)
resample_kernel(const RsRec *__restrict__ recs, int n_rec, const Phase *__restrict__ phases,
                const double *__restrict__ taps, int up, int down, int channels, int tile_out, int s_min, int e_max,
                int span_cap, int16_t *__restrict__ out_all)
{
    using Unit = typename PcmIn<PCM>::Unit;
    constexpr int UNITS = PcmIn<PCM>::UNITS;
    constexpr int VEC = 16 / sizeof(Unit);
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double *xs = reinterpret_cast<double *>(smem_raw);                                   // [span_cap] downmixed frames
    Unit *raw = reinterpret_cast<Unit *>(smem_raw + (((size_t)span_cap * sizeof(double) + 15) & ~(size_t)15));
    const int tid = threadIdx.x;

    int lo = 0, hi = n_rec;                                      // recs[lo].tile_off <= blockIdx.x < recs[hi].tile_off
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (recs[mid].tile_off <= (int64_t)blockIdx.x) lo = mid; else hi = mid; }
    const RsRec &rec = recs[lo];
    const Unit *pcm = reinterpret_cast<const Unit *>(rec.pcm);
    const int64_t fb = rec.f_base, n = rec.n_known;
    const int64_t k0 = rec.k_first + ((int64_t)blockIdx.x - rec.tile_off) * tile_out;
    const int nk = (int)min((int64_t)tile_out, rec.k_first + rec.n_out - k0);
    const int64_t f_lo = (k0 * down) / up + s_min;                            // input frames [f_lo, f_hi)
    const int64_t f_hi = ((k0 + nk - 1) * down) / up + e_max;
    const int span = (int)(f_hi - f_lo);                                      // <= span_cap

    // ---- raw samples of frames [max(f_lo, f_base), min(f_hi, n)); vector loads stay inside the record, since its base
    // is 16-byte aligned and they end at or before unit e_hi ----
    const int64_t g_lo = max(f_lo, fb), g_hi = min(f_hi, n);
    int64_t rb = 0;                                              // raw[i] holds unit rb + i of pcm
    if (g_lo < g_hi) {
        const int64_t e_lo = (g_lo - fb) * channels * UNITS, e_hi = (g_hi - fb) * channels * UNITS;
        if (rec.align == 2) {
            rb = e_lo & ~(int64_t)(VEC - 1);
            const int64_t v_hi = e_hi & ~(int64_t)(VEC - 1);
            const int nv = (int)((v_hi - rb) / VEC);
            const int4 *src = reinterpret_cast<const int4 *>(pcm + rb);
            int4 *dst = reinterpret_cast<int4 *>(raw);
            for (int i = tid; i < nv; i += RS_THREADS) dst[i] = __ldg(src + i);
            for (int64_t e = max(v_hi, rb) + tid; e < e_hi; e += RS_THREADS) raw[e - rb] = pcm[e];
        } else if (sizeof(Unit) == 1 || rec.align == 1) {
            rb = e_lo;
            for (int64_t e = e_lo + tid; e < e_hi; e += RS_THREADS) raw[e - rb] = pcm[e];
        } else {
            rb = e_lo;
            const unsigned char *src = reinterpret_cast<const unsigned char *>(pcm + e_lo);
            unsigned char *dst = reinterpret_cast<unsigned char *>(raw);
            const int64_t nb = (e_hi - e_lo) * (int64_t)sizeof(Unit);
            for (int64_t i = tid; i < nb; i += RS_THREADS) dst[i] = src[i];
        }
    }
    __syncthreads();

    // ---- downmix: mean over the channels in float64, channel order; zeros outside the recording ----
    for (int i = tid; i < span; i += RS_THREADS) {
        const int64_t f = f_lo + i;
        double v = 0.0;
        if (f >= fb && f < n) {
            const Unit *p = raw + ((f - fb) * channels * UNITS - rb);
            double s = 0.0;
            for (int c = 0; c < channels; ++c) s += pcm_value<PCM>(p + c * UNITS);
            v = s / (double)channels;
        }
        xs[i] = v;
    }
    __syncthreads();

    // ---- one float64 dot product per output, taps in ascending frame order ----
    int16_t *out = out_all + rec.out_off;
    for (int j = tid; j < nk; j += RS_THREADS) {
        const int64_t k = k0 + j;
        const int64_t kd = k * down;
        const int64_t a = kd / up;
        const int q = (int)(kd - a * up);
        const Phase ph = phases[q];
        const double *x = xs + (a + ph.s - f_lo);
        const double *t = taps + ph.off;
        double acc = 0.0;
        for (int i = 0; i < ph.n; ++i) acc = fma(__ldg(t + i), x[i], acc);
        const double v = fmin(fmax(rint(acc * 32768.0), -32768.0), 32767.0);     // round half to even, saturate
        out[k - rec.k_first] = (int16_t)(int)v;
    }
}

int gcd_(int a, int b) { while (b) { const int t = a % b; a = b; b = t; } return a; }

bool rate_ok(int rate) { return rate >= RS_MIN_RATE && rate <= RS_MAX_RATE; }

}  // namespace

// One uploaded table: the taps of one (up, down) pair arranged by phase.
struct ResampleTable {
    int up, down;
    int s_min, e_max;               // min s_q, max s_q + n_q over the phases
    Phase *d_phases;
    double *d_taps;
    std::vector<Phase> phases;      // host copy, for the window checks
};

struct ResampleState {
    std::map<int, ResampleTable> tables;      // by input rate
    void *d_recs = nullptr;
    int64_t recs_cap = 0;
};

static ResampleState *rs_state(iss_ctx *ctx)
{
    if (!ctx->resample) ctx->resample = new ResampleState();
    return reinterpret_cast<ResampleState *>(ctx->resample);
}

static void free_table(ResampleTable &t)
{
    if (t.d_phases) cudaFree(t.d_phases);
    if (t.d_taps) cudaFree(t.d_taps);
    t.d_phases = nullptr; t.d_taps = nullptr;
}

void iss_resample_free(iss_ctx *ctx)
{
    if (!ctx->resample) return;
    ResampleState *s = rs_state(ctx);
    for (auto &kv : s->tables) free_table(kv.second);
    if (s->d_recs) cudaFree(s->d_recs);
    delete s;
    ctx->resample = nullptr;
}

extern "C" int64_t iss_resample_num_frames(int64_t n_frames, int rate)
{
    if (!rate_ok(rate) || n_frames < 0) return -1;
    const int g = gcd_(RS_TARGET, rate);
    const int64_t up = RS_TARGET / g, down = rate / g;
    return (n_frames * up + down - 1) / down;
}

extern "C" int iss_resample_upload_taps(iss_ctx *ctx, int rate, const double *h_taps, int64_t n_taps)
{
    ISS_REQUIRE(ctx && h_taps, ISS_ERR_INVALID, "iss_resample_upload_taps: NULL argument");
    ISS_REQUIRE(rate_ok(rate), ISS_ERR_INVALID, "iss_resample_upload_taps: rate %d outside [%d, %d]", rate, RS_MIN_RATE, RS_MAX_RATE);
    const int g = gcd_(RS_TARGET, rate);
    const int up = RS_TARGET / g, down = rate / g;
    const int64_t half = (up == 1 && down == 1) ? 0 : 10 * (int64_t)(up > down ? up : down);
    ISS_REQUIRE(n_taps == 2 * half + 1, ISS_ERR_INVALID,
                "iss_resample_upload_taps: rate %d (up %d, down %d) needs %lld taps, got %lld", rate, up, down,
                (long long)(2 * half + 1), (long long)n_taps);
    ISS_CUDA_OK(cudaSetDevice(ctx->device));
    // Output k with t = k * down + half = m_hi * up + p uses h[p + j * up] against frame m_hi - j while p + j * up <= 2 half.
    // With k * down = a * up + q and half = b * up + r: p = (q + r) mod up and m_hi = a + b + (q + r >= up).
    std::vector<Phase> ph(up);
    std::vector<double> taps;
    taps.reserve((size_t)n_taps);
    const int64_t b = half / up, r = half % up;
    int s_min = 0, e_max = 0;
    for (int q = 0; q < up; ++q) {
        const int64_t carry = (q + r >= up) ? 1 : 0, p = q + r - carry * up;
        const int64_t nq = (2 * half - p) / up + 1;
        Phase &f = ph[q];
        f.off = (int)taps.size(); f.n = (int)nq; f.s = (int)(b + carry - (nq - 1)); f.pad = 0;
        for (int64_t i = 0; i < nq; ++i) taps.push_back(h_taps[p + (nq - 1 - i) * up]);      // ascending frames
        if (q == 0 || f.s < s_min) s_min = f.s;
        if (q == 0 || f.s + f.n > e_max) e_max = f.s + f.n;
    }
    ResampleState *s = rs_state(ctx);
    auto it = s->tables.find(rate);
    if (it != s->tables.end()) { free_table(it->second); s->tables.erase(it); }
    ResampleTable t{up, down, s_min, e_max, nullptr, nullptr, ph};
    cudaError_t e = cudaMalloc(&t.d_phases, sizeof(Phase) * ph.size());
    if (e == cudaSuccess) e = cudaMalloc(&t.d_taps, sizeof(double) * taps.size());
    if (e == cudaSuccess) e = cudaMemcpy(t.d_phases, ph.data(), sizeof(Phase) * ph.size(), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(t.d_taps, taps.data(), sizeof(double) * taps.size(), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        free_table(t);
        iss_set_error("iss_resample_upload_taps: %s", cudaGetErrorString(e));
        return ISS_ERR_CUDA;
    }
    s->tables[rate] = t;
    return ISS_OK;
}

extern "C" int iss_resample_release_taps(iss_ctx *ctx, int rate)
{
    ISS_REQUIRE(ctx, ISS_ERR_INVALID, "iss_resample_release_taps: ctx is NULL");
    if (!ctx->resample) return ISS_OK;
    ISS_CUDA_OK(cudaSetDevice(ctx->device));
    ResampleState *s = rs_state(ctx);
    auto it = s->tables.find(rate);
    if (it != s->tables.end()) { free_table(it->second); s->tables.erase(it); }
    return ISS_OK;
}

// Bytes of one stored sample of a pcm_format check_call accepts.
static int sample_bytes(int pcm_format)
{
    switch (pcm_format) {
    case ISS_PCM_U8: return 1;
    case ISS_PCM_S16: return 2;
    case ISS_PCM_S24: return 3;
    case ISS_PCM_F64: return 8;
    default: return 4;                                   // float32, int32
    }
}

// Largest power-of-two tile (outputs per CTA) whose staged span fits the shared-memory budget.  With 8 channels of
// float64, the widest frame, every rate from 8 to 192 kHz fits at a tile of 64 or more; run_records checks the fit.
static void tile_for(const ResampleTable &t, int channels, int bytes, int *tile, int *span_cap, size_t *smem)
{
    for (int to = RS_MAX_TILE;; to >>= 1) {
        const int64_t span = ((int64_t)(to - 1) * t.down + t.up - 1) / t.up + 1 + (t.e_max - t.s_min);
        const int64_t raw = (span * channels * bytes + 16 + 15) & ~(int64_t)15;           // + one vector of slack
        const int64_t bytes = ((span * (int64_t)sizeof(double) + 15) & ~(int64_t)15) + raw;
        if (bytes <= RS_SMEM_BUDGET || to == RS_MIN_TILE) {
            *tile = to; *span_cap = (int)span; *smem = (size_t)bytes;
            return;
        }
    }
}

template <int PCM>
static int launch_resample(const ResampleTable &t, const RsRec *d_recs, int n_rec, int64_t ntiles, int channels,
                           int tile, int span_cap, size_t smem, int16_t *d_out, cudaStream_t st)
{
    auto kern = resample_kernel<PCM>;
    ISS_CUDA_OK(iss_optin_smem((const void *)kern, (int)smem));
    kern<<<(unsigned)ntiles, RS_THREADS, smem, st>>>(d_recs, n_rec, t.d_phases, t.d_taps, t.up, t.down, channels, tile,
                                                     t.s_min, t.e_max, span_cap, d_out);
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch();
    return ISS_OK;
}

// Checks the common arguments of a resampling call; *out is the table of `rate`.
static int check_call(iss_ctx *ctx, const char *fn, int n_rec, const void *args, int channels, int rate, int pcm_format,
                      const ResampleTable **out)
{
    ISS_REQUIRE(ctx, ISS_ERR_INVALID, "%s: ctx is NULL", fn);
    ISS_REQUIRE(pcm_format == ISS_PCM_F32 || pcm_format == ISS_PCM_S16 || pcm_format == ISS_PCM_U8 ||
                pcm_format == ISS_PCM_S24 || pcm_format == ISS_PCM_S32 || pcm_format == ISS_PCM_F64,
                ISS_ERR_INVALID, "bad pcm_format %d", pcm_format);
    ISS_REQUIRE(channels >= 1 && channels <= RS_MAX_CHANNELS, ISS_ERR_INVALID,
                "%s: %d channels outside [1, %d]", fn, channels, RS_MAX_CHANNELS);
    ISS_REQUIRE(rate_ok(rate), ISS_ERR_INVALID, "%s: rate %d outside [%d, %d]", fn, rate, RS_MIN_RATE, RS_MAX_RATE);
    ISS_REQUIRE(n_rec >= 1 && args, ISS_ERR_INVALID, "%s: bad argument", fn);
    ResampleState *s = rs_state(ctx);
    auto it = s->tables.find(rate);
    ISS_REQUIRE(it != s->tables.end(), ISS_ERR_STATE, "%s: no taps uploaded for rate %d", fn, rate);
    *out = &it->second;
    return ISS_OK;
}

// Tiles the records (recs[0 .. n_rec), pcm .. out_off set), uploads the record table and launches.
static int run_records(iss_ctx *ctx, const char *fn, const ResampleTable &t, std::vector<RsRec> &recs, int channels,
                       int pcm_format, int16_t *d_out, void *stream)
{
    ResampleState *s = rs_state(ctx);
    ISS_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = iss_stream(stream);
    int tile, span_cap;
    size_t smem;
    tile_for(t, channels, sample_bytes(pcm_format), &tile, &span_cap, &smem);
    const uintptr_t unit = pcm_format == ISS_PCM_S24 ? 1 : (uintptr_t)sample_bytes(pcm_format);     // bytes of a Unit
    ISS_REQUIRE(smem <= (size_t)RS_SMEM_BUDGET, ISS_ERR_INVALID, "%s: staged span of %zu bytes over the budget", fn, smem);
    const int n_rec = (int)recs.size() - 1;
    int64_t ntiles = 0;
    for (int i = 0; i < n_rec; ++i) {
        RsRec &r = recs[i];
        r.tile_off = ntiles;
        const uintptr_t a = reinterpret_cast<uintptr_t>(r.pcm);
        r.align = (a & 15) == 0 ? 2 : (a % unit == 0 ? 1 : 0);
        ntiles += (r.n_out + tile - 1) / tile;
    }
    recs[n_rec] = RsRec{nullptr, 0, 0, 0, 0, 0, ntiles, 0};
    if (ntiles == 0) return ISS_OK;
    ISS_REQUIRE(d_out, ISS_ERR_INVALID, "%s: NULL output", fn);
    ISS_REQUIRE(ntiles < (1ll << 31), ISS_ERR_INVALID, "%s: input too long for one call", fn);
    if (n_rec + 1 > s->recs_cap) {
        if (s->d_recs) ISS_CUDA_OK(cudaFree(s->d_recs));
        s->d_recs = nullptr; s->recs_cap = 0;
        const int64_t cap = n_rec + 1 + n_rec / 2 + 64;
        cudaError_t e = cudaMalloc(&s->d_recs, (size_t)cap * sizeof(RsRec));
        if (e != cudaSuccess) { iss_set_error("cudaMalloc recording table: %s", cudaGetErrorString(e)); return ISS_ERR_NOMEM; }
        s->recs_cap = cap;
    }
    const RsRec *d_recs = reinterpret_cast<const RsRec *>(s->d_recs);
    ISS_CUDA_OK(cudaMemcpyAsync(s->d_recs, recs.data(), sizeof(RsRec) * (n_rec + 1), cudaMemcpyHostToDevice, st));
    switch (pcm_format) {
    case ISS_PCM_S16: return launch_resample<ISS_PCM_S16>(t, d_recs, n_rec, ntiles, channels, tile, span_cap, smem, d_out, st);
    case ISS_PCM_U8: return launch_resample<ISS_PCM_U8>(t, d_recs, n_rec, ntiles, channels, tile, span_cap, smem, d_out, st);
    case ISS_PCM_S24: return launch_resample<ISS_PCM_S24>(t, d_recs, n_rec, ntiles, channels, tile, span_cap, smem, d_out, st);
    case ISS_PCM_S32: return launch_resample<ISS_PCM_S32>(t, d_recs, n_rec, ntiles, channels, tile, span_cap, smem, d_out, st);
    case ISS_PCM_F64: return launch_resample<ISS_PCM_F64>(t, d_recs, n_rec, ntiles, channels, tile, span_cap, smem, d_out, st);
    default: return launch_resample<ISS_PCM_F32>(t, d_recs, n_rec, ntiles, channels, tile, span_cap, smem, d_out, st);
    }
}

extern "C" int iss_resample_to16k_multi(iss_ctx *ctx, int n_rec, const void *const *h_pcm, const int64_t *h_n_frames,
                                        int channels, int rate, int pcm_format, int16_t *d_out, const int64_t *h_out_off,
                                        void *stream)
{
    const char *fn = "iss_resample_to16k_multi";
    const ResampleTable *t = nullptr;
    const int rc = check_call(ctx, fn, n_rec, h_pcm && h_n_frames && h_out_off ? h_pcm : nullptr, channels, rate,
                              pcm_format, &t);
    if (rc != ISS_OK) return rc;
    std::vector<RsRec> recs(n_rec + 1);
    for (int i = 0; i < n_rec; ++i) {
        RsRec &r = recs[i];
        r.pcm = h_pcm[i];
        r.f_base = 0;
        r.n_known = h_n_frames[i];
        ISS_REQUIRE(r.n_known >= 0 && r.n_known < ((int64_t)1 << 40), ISS_ERR_INVALID,
                    "iss_resample_to16k_multi: bad frame count (recording %d)", i);
        r.k_first = 0;
        r.n_out = iss_resample_num_frames(r.n_known, rate);
        r.out_off = h_out_off[i];
        ISS_REQUIRE(r.n_out == 0 || r.pcm, ISS_ERR_INVALID, "iss_resample_to16k_multi: NULL buffer (recording %d)", i);
        ISS_REQUIRE(r.out_off >= 0, ISS_ERR_INVALID, "iss_resample_to16k_multi: negative offset (recording %d)", i);
    }
    return run_records(ctx, fn, *t, recs, channels, pcm_format, d_out, stream);
}

extern "C" int iss_resample_window_multi(iss_ctx *ctx, int n_rec, const void *const *h_pcm, const int64_t *h_win,
                                         int channels, int rate, int pcm_format, int16_t *d_out, void *stream)
{
    const char *fn = "iss_resample_window_multi";
    const ResampleTable *t = nullptr;
    const int rc = check_call(ctx, fn, n_rec, h_pcm && h_win ? h_pcm : nullptr, channels, rate, pcm_format, &t);
    if (rc != ISS_OK) return rc;
    const int64_t up = t->up, down = t->down;
    std::vector<RsRec> recs(n_rec + 1);
    for (int i = 0; i < n_rec; ++i) {
        const int64_t *w = h_win + (size_t)i * 6;
        const int64_t f_base = w[0], n_known = w[1], k_first = w[2], n_out = w[3], out_off = w[4], flags = w[5];
        ISS_REQUIRE(f_base >= 0 && f_base <= n_known && n_known < ((int64_t)1 << 40) && k_first >= 0 &&
                    k_first < ((int64_t)1 << 44) && n_out >= 0 && n_out < ((int64_t)1 << 44) && out_off >= 0 && (flags & ~(int64_t)ISS_RESAMPLE_END) == 0, ISS_ERR_INVALID,
                    "%s: record %d: bad field", fn, i);
        ISS_REQUIRE(k_first + n_out <= iss_resample_num_frames(n_known, rate), ISS_ERR_INVALID,
                    "%s: record %d: outputs [%lld, %lld) past the %lld outputs of %lld frames", fn, i,
                    (long long)k_first, (long long)(k_first + n_out), (long long)iss_resample_num_frames(n_known, rate),
                    (long long)n_known);
        ISS_REQUIRE(n_out == 0 || h_pcm[i], ISS_ERR_INVALID, "%s: record %d: NULL buffer", fn, i);
        if (n_out > 0) {
            // the frames an output reads, a + s_q .. a + s_q + n_q - 1, move forward with k: the first and last
            // output bound the window
            const int64_t k_last = k_first + n_out - 1;
            const int64_t a0 = k_first * down / up, a1 = k_last * down / up;
            const Phase &p0 = t->phases[(size_t)(k_first * down - a0 * up)];
            const Phase &p1 = t->phases[(size_t)(k_last * down - a1 * up)];
            const int64_t first = a0 + p0.s, last = a1 + p1.s + p1.n - 1;
            ISS_REQUIRE(f_base == 0 || first >= f_base, ISS_ERR_INVALID,
                        "%s: record %d: output %lld reads frame %lld, before the window's first frame %lld", fn, i,
                        (long long)k_first, (long long)first, (long long)f_base);
            ISS_REQUIRE((flags & ISS_RESAMPLE_END) || last < n_known, ISS_ERR_INVALID,
                        "%s: record %d: output %lld reads frame %lld of %lld known frames, and the stream has not ended",
                        fn, i, (long long)k_last, (long long)last, (long long)n_known);
        }
        recs[i] = RsRec{h_pcm[i], f_base, n_known, k_first, n_out, out_off, 0, 0};
    }
    return run_records(ctx, fn, *t, recs, channels, pcm_format, d_out, stream);
}
