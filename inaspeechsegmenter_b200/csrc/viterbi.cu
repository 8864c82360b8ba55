// viterbi.cu -- K3: max-sum Viterbi smoothing on device.
//
// Reference semantics: inaSpeechSegmenter/pyannote_viterbi.py:118-224 as called
// from segmenter.py:72 (energy, K = 2) and :176 (CNN posteriors, K = 2 or 3):
//   V[0,j] = E[0,j] + log(1/K);  P[t,j] = first argmax_k (V[t-1,k] + A[k,j]);
//   V[t,j] = E[t,j] + (V[t-1,P] + A[P,j]);  backtrack from first argmax V[T-1].
//
// Exactness: the forward recursion is evaluated in IEEE double in exactly the
// reference's order of operations (so every argmax decision sees the same bits);
// that chain is inherently serial, so the forward pass runs one warp per
// sequence: the 32 lanes fetch and convert 32 steps of emissions in parallel
// (coalesced), then replay them through register shuffles while every lane
// carries the same V; lane j keeps step j's back-pointer byte so stores are
// coalesced too.  The backtrack -- pure integer function composition, hence
// associative and exact -- is parallel: per-256-step chunk maps, a short serial
// scan over chunk maps, then all chunks emit their states concurrently.
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <vector>

#include "iss_common.cuh"

namespace {

constexpr int CH = 256;            // backtrack chunk (steps)
constexpr int MAXK = 4;

struct VitParams {
    double A[MAXK][MAXK];          // from -> to
    double prior;
    double emis_hit, emis_miss;    // energy mode
    double log_ratio;
};

struct VitLayout {
    uint8_t *bp;                   // [total] one byte per step: 2 bits per destination state
    uint8_t *cmap;                 // [nchunks] composite map per chunk
    uint8_t *cend;                 // [nchunks] state at the last step of each chunk
    int64_t *seg_off;              // [n_seg+1]
    int64_t *chunk_off;            // [n_seg+1]
    uint8_t *last;                 // [n_seg] argmax V[T-1]
    // partial-chain support (time-sharded recordings)
    const double *vin;             // [n_seg][MAXK] incoming scores (continue from a predecessor) or nullptr
    double *vout;                  // [n_seg][MAXK] outgoing scores V[T-1] or nullptr
    int alias;                     // 1: every block walks the SAME range seg_off[0..1] (basis chains of a transfer matrix)
                                   // 2: block b walks segment b / 2 with vin / vout slot b (two basis chains per segment)
    int store_bp;                  // 0: scores only
    int stats_stride;              // energy mode: sequence s thresholds on stats[s * stats_stride ..] (0: one shared pair)
    const int64_t *out_off;        // [n_seg] first output of each sequence when out_stride > 1, or nullptr (single sequence)
};

__device__ __forceinline__ bool better(double c, double best)
{
    // numpy.argmax: strictly greater replaces; the first NaN wins and sticks.
    return !(c <= best) && (best == best);
}

// np.mean(f32 array) is f32; + np.log(ratio) (f64) promotes to f64 (segmenter.py:70).  sg = {sum, count}.
__device__ __forceinline__ double energy_threshold(const double *sg, double log_ratio)
{
    const double cnt = sg[1];
    const float mean32 = (float)(sg[0] / cnt);          // 0/0 -> NaN like the mean of an empty slice
    return (double)mean32 + log_ratio;
}

// emissions of step `i` of src: loge against thr (energy) or log(p) of posterior row i
template <int K, bool ENERGY>
__device__ __forceinline__ void load_emissions(const float *__restrict__ src, int64_t i, double thr, const VitParams &prm,
                                               double (&e)[K])
{
    if (ENERGY) {
        const bool raw = (double)src[i] > thr;          // NaN thr -> all false
        e[0] = raw ? prm.emis_miss : prm.emis_hit;
        e[1] = raw ? prm.emis_hit : prm.emis_miss;
    } else {
#pragma unroll
        for (int j = 0; j < K; ++j)                     // np.log on float32, correctly rounded
            e[j] = (double)(float)log((double)src[i * K + j]);
    }
}

// one DP step on emissions `es`; `is_first` only for the very first step of the sequence.  Returns the step's
// back-pointers, 2 bits per destination state.
template <int K, bool ENERGY>
__device__ __forceinline__ unsigned vit_step(double (&V)[K], const double (&es)[K], const VitParams &prm, bool is_first)
{
    unsigned bp = 0;
    if (is_first) {
#pragma unroll
        for (int j = 0; j < K; ++j) { V[j] = es[j] + prm.prior; bp |= (unsigned)j << (2 * j); }
    } else {
        double Vn[K];
#pragma unroll
        for (int j = 0; j < K; ++j) {
            double best = V[0] + prm.A[0][j];
            double vn = es[j] + best;
            unsigned arg = 0;
#pragma unroll
            for (int k = 1; k < K; ++k) {
                const double c = V[k] + prm.A[k][j];
                const double vc = es[j] + c;            // speculative: same op whichever wins
                // energy emissions / transitions are finite constants: V can never be NaN there
                const bool u = ENERGY ? (c > best) : better(c, best);
                best = u ? c : best;
                vn = u ? vc : vn;
                arg = u ? (unsigned)k : arg;
            }
            Vn[j] = vn;
            bp |= arg << (2 * j);
        }
#pragma unroll
        for (int j = 0; j < K; ++j) V[j] = Vn[j];
    }
    return bp;
}

// first argmax (numpy.argmax, NaN rule of better())
template <int K>
__device__ __forceinline__ int first_argmax(const double (&V)[K])
{
    int arg = 0;
    double best = V[0];
#pragma unroll
    for (int k = 1; k < K; ++k) {
        const bool u = better(V[k], best);
        best = u ? V[k] : best;
        arg = u ? k : arg;
    }
    return arg;
}

// composition of back-pointer maps: (f o m)[x] = f[m[x]], 2-bit fields
__device__ __forceinline__ unsigned compose_map(unsigned f, unsigned m)
{
    unsigned r = 0;
#pragma unroll
    for (int x = 0; x < 4; ++x) r |= ((f >> (2 * ((m >> (2 * x)) & 3))) & 3) << (2 * x);
    return r;
}

template <int K, bool ENERGY>
__global__ void __launch_bounds__(32)
viterbi_forward_kernel(const float *__restrict__ src, const double *__restrict__ stats, VitParams prm, VitLayout lay)
{
    const int slot = blockIdx.x, lane = threadIdx.x;             // slot indexes vin / vout / last
    const int seg = lay.alias == 1 ? 0 : (lay.alias == 2 ? slot >> 1 : slot);
    const int64_t t0 = lay.seg_off[seg];
    const int64_t T = lay.seg_off[seg + 1] - t0;
    if (T <= 0) return;
    const bool cont = lay.vin != nullptr;          // first step is an ordinary transition from vin
    const double thr = ENERGY ? energy_threshold(stats + (int64_t)seg * lay.stats_stride, prm.log_ratio) : 0.0;
    double V[K];
#pragma unroll
    for (int j = 0; j < K; ++j) V[j] = cont ? lay.vin[slot * MAXK + j] : 0.0;

    for (int64_t base = 0; base < T; base += 32) {
        const int64_t t = base + lane;
        double e[K];
#pragma unroll
        for (int j = 0; j < K; ++j) e[j] = 0.0;
        if (t < T) load_emissions<K, ENERGY>(src, t0 + t, thr, prm, e);
        const int nstep = (int)min((int64_t)32, T - base);
        unsigned mybp = 0;
        auto dp_step = [&](const double (&es)[K], bool is_first) -> unsigned { return vit_step<K, ENERGY>(V, es, prm, is_first); };
        if (nstep == 32 && (base > 0 || cont)) {
            // full block, fully unrolled: the 32 x K emission shuffles do not depend on V, so they are
            // issued ahead and only the add/compare/select chain remains on the serial critical path
#pragma unroll
            for (int s = 0; s < 32; ++s) {
                double es[K];
#pragma unroll
                for (int j = 0; j < K; ++j) es[j] = __shfl_sync(0xffffffffu, e[j], s);
                const unsigned bp = dp_step(es, false);
                mybp = (lane == s) ? bp : mybp;
            }
        } else {
            for (int s = 0; s < nstep; ++s) {
                double es[K];
#pragma unroll
                for (int j = 0; j < K; ++j) es[j] = __shfl_sync(0xffffffffu, e[j], s);
                const unsigned bp = dp_step(es, base + s == 0 && !cont);
                if (lane == s) mybp = bp;
            }
        }
        if (t < T && lay.store_bp) lay.bp[t0 + t] = (uint8_t)mybp;
    }
    if (lane == 0) {
        const int arg = first_argmax<K>(V);
        if (lay.store_bp) lay.last[slot] = (uint8_t)arg;
        if (lay.vout) {
#pragma unroll
            for (int k = 0; k < K; ++k) lay.vout[slot * MAXK + k] = V[k];
        }
    }
}

__device__ __forceinline__ int find_seg(const int64_t *chunk_off, int n_seg, int64_t c)
{
    int lo = 0, hi = n_seg;            // chunk_off[lo] <= c < chunk_off[hi]
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (chunk_off[mid] <= c) lo = mid; else hi = mid;
    }
    return lo;
}

// cmap[c]: (state at the last step of chunk c) -> (state at the last step of chunk c-1)
__global__ void viterbi_chunk_map_kernel(VitLayout lay, int n_seg, int64_t nchunks, int has_pred)
{
    const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nchunks) return;
    const int seg = find_seg(lay.chunk_off, n_seg, c);
    const int64_t t0 = lay.seg_off[seg], T = lay.seg_off[seg + 1] - t0;
    const int64_t lc = c - lay.chunk_off[seg];
    const int64_t a = lc * CH, b = min(a + CH, T);          // steps [a, b)
    unsigned m = 0xE4;                                      // identity: 3,2,1,0 in 2-bit fields
    const uint8_t *bp = lay.bp + t0;
    for (int64_t t = b - 1; t >= a; --t) {
        if (t == 0 && !has_pred) break;                     // bp[0] is unused when the sequence has no predecessor
        const unsigned f = bp[t];
        unsigned r = 0;
#pragma unroll
        for (int x = 0; x < 4; ++x) r |= ((f >> (2 * ((m >> (2 * x)) & 3))) & 3) << (2 * x);
        m = r;
    }
    lay.cmap[c] = (uint8_t)m;
}

// serial over the chunks of one segment (T/256 steps), one thread per segment
__global__ void viterbi_chunk_scan_kernel(VitLayout lay, int n_seg)
{
    const int seg = blockIdx.x * blockDim.x + threadIdx.x;
    if (seg >= n_seg) return;
    const int64_t c0 = lay.chunk_off[seg], c1 = lay.chunk_off[seg + 1];
    if (c1 <= c0) return;
    unsigned x = lay.last[seg];
    for (int64_t c = c1 - 1; c >= c0; --c) {
        lay.cend[c] = (uint8_t)x;
        x = (lay.cmap[c] >> (2 * x)) & 3;
    }
}

__global__ void viterbi_chunk_emit_kernel(VitLayout lay, int n_seg, int64_t nchunks, int out_stride,
                                          uint8_t *__restrict__ states)
{
    const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nchunks) return;
    const int seg = find_seg(lay.chunk_off, n_seg, c);
    const int64_t t0 = lay.seg_off[seg], T = lay.seg_off[seg + 1] - t0;
    const int64_t lc = c - lay.chunk_off[seg];
    const int64_t a = lc * CH, b = min(a + CH, T);
    const uint8_t *bp = lay.bp + t0;
    unsigned x = lay.cend[c];
    const int64_t o0 = lay.out_off ? lay.out_off[seg] : t0;         // a single sequence has t0 == 0
    for (int64_t t = b - 1; t >= a; --t) {
        if (out_stride == 1) states[o0 + t] = (uint8_t)x;
        else if (t % out_stride == 0) states[o0 + t / out_stride] = (uint8_t)x;
        x = (bp[t] >> (2 * x)) & 3;
    }
}

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

struct HostPlan {
    std::vector<int64_t> seg_off, chunk_off;
    int64_t total, nchunks;
};

int make_layout(const int64_t *h_seg_off, int n_seg, void *d_work, HostPlan &hp, VitLayout &lay, cudaStream_t st)
{
    hp.seg_off.assign(h_seg_off, h_seg_off + n_seg + 1);
    hp.chunk_off.resize(n_seg + 1);
    int64_t nc = 0;
    for (int s = 0; s < n_seg; ++s) {
        hp.chunk_off[s] = nc;
        const int64_t T = h_seg_off[s + 1] - h_seg_off[s];
        ISS_REQUIRE(T >= 0, ISS_ERR_INVALID, "viterbi: segment offsets must be non-decreasing");
        nc += (T + CH - 1) / CH;
    }
    hp.chunk_off[n_seg] = nc;
    hp.total = h_seg_off[n_seg];
    hp.nchunks = nc;
    uint8_t *p = reinterpret_cast<uint8_t *>(d_work);
    size_t o = 0;
    lay.bp = p + o;        o = align_up(o + (size_t)hp.total, 256);
    lay.cmap = p + o;      o = align_up(o + (size_t)nc, 256);
    lay.cend = p + o;      o = align_up(o + (size_t)nc, 256);
    lay.seg_off = reinterpret_cast<int64_t *>(p + o);   o = align_up(o + sizeof(int64_t) * (n_seg + 1), 256);
    lay.chunk_off = reinterpret_cast<int64_t *>(p + o); o = align_up(o + sizeof(int64_t) * (n_seg + 1), 256);
    lay.last = p + o;
    ISS_CUDA_OK(cudaMemcpyAsync(lay.seg_off, hp.seg_off.data(), sizeof(int64_t) * (n_seg + 1), cudaMemcpyHostToDevice, st));
    ISS_CUDA_OK(cudaMemcpyAsync(lay.chunk_off, hp.chunk_off.data(), sizeof(int64_t) * (n_seg + 1), cudaMemcpyHostToDevice, st));
    return ISS_OK;
}

int run_backtrack(const VitLayout &lay, const HostPlan &hp, int n_seg, int out_stride, uint8_t *d_states, cudaStream_t st)
{
    if (hp.nchunks == 0) return ISS_OK;
    const int TB = 128;
    const unsigned gc = (unsigned)((hp.nchunks + TB - 1) / TB);
    viterbi_chunk_map_kernel<<<gc, TB, 0, st>>>(lay, n_seg, hp.nchunks, 0);
    viterbi_chunk_scan_kernel<<<(n_seg + 63) / 64, 64, 0, st>>>(lay, n_seg);
    viterbi_chunk_emit_kernel<<<gc, TB, 0, st>>>(lay, n_seg, hp.nchunks, out_stride, d_states);
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch(3);
    return ISS_OK;
}

// composite of all chunk maps of sequence 0: (state at the last step) -> (state just before the first step)
__global__ void viterbi_compose_kernel(VitLayout lay, int64_t nchunks, uint8_t *out)
{
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    unsigned m = 0xE4;
    for (int64_t c = nchunks - 1; c >= 0; --c) {
        const unsigned f = lay.cmap[c];
        unsigned r = 0;
#pragma unroll
        for (int x = 0; x < 4; ++x) r |= ((f >> (2 * ((m >> (2 * x)) & 3))) & 3) << (2 * x);
        m = r;
    }
    out[0] = (uint8_t)m;
}

__global__ void viterbi_set_last_kernel(VitLayout lay, int state) { if (threadIdx.x == 0 && blockIdx.x == 0) lay.last[0] = (uint8_t)state; }

}  // namespace

// ---- partial chains of the energy Viterbi for time-sharded recordings (SURVEY 8(e)) -------------------
static void fill_energy_params(VitParams &prm, const double *h_emis, const double *h_trans, double log_prior, double log_ratio)
{
    for (int i = 0; i < 2; ++i) for (int j = 0; j < 2; ++j) prm.A[i][j] = h_trans[i * 2 + j];
    prm.prior = log_prior; prm.emis_hit = h_emis[0]; prm.emis_miss = h_emis[1]; prm.log_ratio = log_ratio;
}

extern "C" int iss_energy_transfer(iss_ctx *ctx, const float *d_loge, int64_t L, const double *d_loge_stats,
                                   double log_ratio, const double *h_emis, const double *h_trans,
                                   double *h_matrix, void *d_work, void *stream)
{
    ISS_REQUIRE(ctx && d_loge && d_loge_stats && h_emis && h_trans && h_matrix && d_work && L > 0, ISS_ERR_INVALID, "iss_energy_transfer: bad argument");
    ISS_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = iss_stream(stream);
    const int64_t off[2] = {0, L};
    HostPlan hp; VitLayout lay = {};
    int rc = make_layout(off, 1, d_work, hp, lay, st);
    if (rc != ISS_OK) return rc;
    // scratch for vin / vout lives behind `last`
    double *d_v = reinterpret_cast<double *>(lay.last + 256);
    const double NEG_INF = -INFINITY;
    double vin[2 * MAXK] = {0.0, NEG_INF, 0, 0, NEG_INF, 0.0, 0, 0};      // basis vectors e_0, e_1 (max-plus)
    ISS_CUDA_OK(cudaMemcpyAsync(d_v, vin, sizeof(vin), cudaMemcpyHostToDevice, st));
    lay.vin = d_v; lay.vout = d_v + 2 * MAXK; lay.alias = 1; lay.store_bp = 0;
    VitParams prm = {};
    fill_energy_params(prm, h_emis, h_trans, 0.0, log_ratio);
    viterbi_forward_kernel<2, true><<<2, 32, 0, st>>>(d_loge, d_loge_stats, prm, lay);
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch();
    double vout[2 * MAXK];
    ISS_CUDA_OK(cudaMemcpyAsync(vout, lay.vout, sizeof(vout), cudaMemcpyDeviceToHost, st));
    ISS_CUDA_OK(cudaStreamSynchronize(st));
    // M[j][i] = score of ending in j having started (before the first frame) in i
    for (int i = 0; i < 2; ++i) for (int j = 0; j < 2; ++j) h_matrix[j * 2 + i] = vout[i * MAXK + j];
    return ISS_OK;
}

extern "C" int iss_energy_forward(iss_ctx *ctx, const float *d_loge, int64_t L, const double *d_loge_stats,
                                  double log_ratio, const double *h_emis, const double *h_trans, double log_prior,
                                  const double *h_vin, double *h_vout, uint8_t *h_backmap, void *d_work, void *stream)
{
    ISS_REQUIRE(ctx && d_loge && d_loge_stats && h_emis && h_trans && h_vout && h_backmap && d_work && L > 0, ISS_ERR_INVALID, "iss_energy_forward: bad argument");
    ISS_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = iss_stream(stream);
    const int64_t off[2] = {0, L};
    HostPlan hp; VitLayout lay = {};
    int rc = make_layout(off, 1, d_work, hp, lay, st);
    if (rc != ISS_OK) return rc;
    double *d_v = reinterpret_cast<double *>(lay.last + 256);
    if (h_vin) {
        double vin[MAXK] = {h_vin[0], h_vin[1], 0, 0};
        ISS_CUDA_OK(cudaMemcpyAsync(d_v, vin, sizeof(vin), cudaMemcpyHostToDevice, st));
        lay.vin = d_v;
    }
    lay.vout = d_v + 2 * MAXK; lay.alias = 0; lay.store_bp = 1;
    VitParams prm = {};
    fill_energy_params(prm, h_emis, h_trans, log_prior, log_ratio);
    viterbi_forward_kernel<2, true><<<1, 32, 0, st>>>(d_loge, d_loge_stats, prm, lay);
    const unsigned gc = (unsigned)((hp.nchunks + 127) / 128);
    viterbi_chunk_map_kernel<<<gc, 128, 0, st>>>(lay, 1, hp.nchunks, h_vin ? 1 : 0);
    uint8_t *d_map = reinterpret_cast<uint8_t *>(d_v + 4 * MAXK);
    viterbi_compose_kernel<<<1, 32, 0, st>>>(lay, hp.nchunks, d_map);
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch(3);
    double vout[MAXK];
    uint8_t m;
    ISS_CUDA_OK(cudaMemcpyAsync(vout, lay.vout, sizeof(vout), cudaMemcpyDeviceToHost, st));
    ISS_CUDA_OK(cudaMemcpyAsync(&m, d_map, 1, cudaMemcpyDeviceToHost, st));
    ISS_CUDA_OK(cudaStreamSynchronize(st));
    h_vout[0] = vout[0]; h_vout[1] = vout[1];
    h_backmap[0] = m & 3; h_backmap[1] = (m >> 2) & 3;
    return ISS_OK;
}

extern "C" int iss_energy_emit(iss_ctx *ctx, int64_t L, int end_state, int out_stride, uint8_t *d_states,
                               void *d_work, void *stream)
{
    ISS_REQUIRE(ctx && d_states && d_work && L > 0 && out_stride >= 1 && end_state >= -1 && end_state < 2, ISS_ERR_INVALID, "iss_energy_emit: bad argument");
    ISS_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = iss_stream(stream);
    // same carve as iss_energy_forward (no copies: the tables are already on the device)
    HostPlan hp; VitLayout lay = {};
    hp.seg_off = {0, L}; hp.chunk_off = {0, (L + CH - 1) / CH}; hp.total = L; hp.nchunks = (L + CH - 1) / CH;
    uint8_t *p = reinterpret_cast<uint8_t *>(d_work);
    size_t o = 0;
    lay.bp = p + o;        o = align_up(o + (size_t)hp.total, 256);
    lay.cmap = p + o;      o = align_up(o + (size_t)hp.nchunks, 256);
    lay.cend = p + o;      o = align_up(o + (size_t)hp.nchunks, 256);
    lay.seg_off = reinterpret_cast<int64_t *>(p + o);   o = align_up(o + sizeof(int64_t) * 2, 256);
    lay.chunk_off = reinterpret_cast<int64_t *>(p + o); o = align_up(o + sizeof(int64_t) * 2, 256);
    lay.last = p + o;
    if (end_state >= 0) viterbi_set_last_kernel<<<1, 32, 0, st>>>(lay, end_state);
    const unsigned gc = (unsigned)((hp.nchunks + 127) / 128);
    viterbi_chunk_scan_kernel<<<1, 64, 0, st>>>(lay, 1);
    viterbi_chunk_emit_kernel<<<gc, 128, 0, st>>>(lay, 1, hp.nchunks, out_stride, d_states);
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch(3);
    return ISS_OK;
}

// ---- chunk-parallel energy Viterbi ------------------------------------------------------------------------
// The whole-file chain (3.6 M frames per 10 h, ~40 ns per frame when walked serially = 6-9 % of a step) is cut
// into chunks of ECH frames that are walked CONCURRENTLY, exactly as shard.py cuts it at rank boundaries:
//   1. chunk 0: its true forward pass (scores out);  chunks 1..C-1: the 2x2 max-plus transfer matrix of the
//      chunk (two basis-vector chains per chunk)                                    -- 2C - 1 concurrent chains
//   2. one thread composes the entry scores  entry[c+1][j] = max_i(entry[c][i] + M_c[j][i])
//   3. chunks 1..C-1: true forward pass from their entry scores (back-pointers stored)   -- C - 1 chains
//   4. the usual parallel backtrack over the whole sequence.
// Exact in exact arithmetic; in IEEE double the entry scores are associated differently from the serial chain
// (one addition of a chunk-relative score instead of ECH stepwise additions), which could only matter for a
// path tie closer than ~1e-8 -- the path scores are sums of a handful of constants (-5, -345.39, -23.03, -1e-10)
// whose distinct combinations are orders of magnitude further apart.  The serial kernel stays available
// (ISS_B200_VITERBI=serial, and it is what the GPU tests compare this against on 10 h tracks).
constexpr int64_t ECH = 16384;

__global__ void energy_entry_compose_kernel(const double *__restrict__ v0, const double *__restrict__ basis_out,
                                            int nchunk, double *__restrict__ entry)
{
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    double e0 = v0[0], e1 = v0[1];                               // scores leaving chunk 0 = entering chunk 1
    for (int c = 1; c < nchunk; ++c) {
        entry[(c - 1) * MAXK + 0] = e0; entry[(c - 1) * MAXK + 1] = e1;
        // basis_out slot 2(c-1)+i = scores leaving chunk c when entering in state i with score 0
        const double *m0 = basis_out + (size_t)(2 * (c - 1)) * MAXK, *m1 = m0 + MAXK;
        const double a0 = e0 + m0[0], b0 = e1 + m1[0], a1 = e0 + m0[1], b1 = e1 + m1[1];
        e0 = (b0 > a0) ? b0 : a0;
        e1 = (b1 > a1) ? b1 : a1;
    }
}

static int g_energy_serial = -1;        // -1: read ISS_B200_VITERBI on first use
static bool energy_serial()
{
    if (g_energy_serial < 0) { const char *e = getenv("ISS_B200_VITERBI"); g_energy_serial = (e && !strcmp(e, "serial")) ? 1 : 0; }
    return g_energy_serial == 1;
}
extern "C" int iss_set_energy_viterbi_serial(int serial) { g_energy_serial = serial ? 1 : 0; return ISS_OK; }

static int energy_viterbi_chunked(iss_ctx *ctx, const float *d_loge, int64_t L, const double *d_loge_stats, const VitParams &prm,
                                  int out_stride, uint8_t *d_states, void *d_work, cudaStream_t st)
{
    const int C = (int)((L + ECH - 1) / ECH);
    // backtrack layout: ONE sequence [0, L)
    const int64_t off1[2] = {0, L};
    HostPlan hp1; VitLayout lay1 = {};
    int rc = make_layout(off1, 1, d_work, hp1, lay1, st);
    if (rc != ISS_OK) return rc;
    // forward layout: C segments over the same back-pointer array, tables behind lay1's
    uint8_t *p = lay1.last + 256;
    size_t o = 0;
    std::vector<int64_t> seg(C + 1);
    for (int c = 0; c <= C; ++c) seg[c] = std::min<int64_t>((int64_t)c * ECH, L);
    VitLayout lay = lay1;
    lay.seg_off = reinterpret_cast<int64_t *>(p + o); o = align_up(o + sizeof(int64_t) * (C + 1), 256);
    lay.last = p + o;                                  o = align_up(o + (size_t)2 * C, 256);
    double *d_v0 = reinterpret_cast<double *>(p + o);  o += sizeof(double) * MAXK;
    double *d_basis_in = reinterpret_cast<double *>(p + o);  o += sizeof(double) * MAXK * 2 * C;
    double *d_basis_out = reinterpret_cast<double *>(p + o); o += sizeof(double) * MAXK * 2 * C;
    double *d_entry = reinterpret_cast<double *>(p + o);     o += sizeof(double) * MAXK * C;
    ISS_CUDA_OK(cudaMemcpyAsync(lay.seg_off, seg.data(), sizeof(int64_t) * (C + 1), cudaMemcpyHostToDevice, st));
    std::vector<double> basis((size_t)MAXK * 2 * C, 0.0);
    for (int c = 0; c < C; ++c) {                                // e_0 = (0, -inf), e_1 = (-inf, 0) in max-plus
        basis[(size_t)(2 * c) * MAXK + 1] = -INFINITY;
        basis[(size_t)(2 * c + 1) * MAXK + 0] = -INFINITY;
    }
    ISS_CUDA_OK(cudaMemcpyAsync(d_basis_in, basis.data(), sizeof(double) * basis.size(), cudaMemcpyHostToDevice, st));
    // 1a. chunk 0, true pass (prior on the first frame), back-pointers stored
    VitLayout l0 = lay; l0.vin = nullptr; l0.vout = d_v0; l0.alias = 0; l0.store_bp = 1;
    viterbi_forward_kernel<2, true><<<1, 32, 0, st>>>(d_loge, d_loge_stats, prm, l0);
    // 1b. chunks 1..C-1: two basis chains each (segment index = 1 + slot / 2 => shift the offset table by one)
    VitLayout lb = lay; lb.seg_off = lay.seg_off + 1; lb.vin = d_basis_in; lb.vout = d_basis_out; lb.alias = 2; lb.store_bp = 0;
    viterbi_forward_kernel<2, true><<<2 * (C - 1), 32, 0, st>>>(d_loge, d_loge_stats, prm, lb);
    // 2. entry scores of chunks 1..C-1
    energy_entry_compose_kernel<<<1, 32, 0, st>>>(d_v0, d_basis_out, C, d_entry);
    // 3. chunks 1..C-1, true pass from their entry scores
    VitLayout lt = lay; lt.seg_off = lay.seg_off + 1; lt.vin = d_entry; lt.vout = nullptr; lt.alias = 0; lt.store_bp = 1;
    lt.last = lay.last + 1;                                      // last[c] = argmax V at the end of chunk c
    viterbi_forward_kernel<2, true><<<C - 1, 32, 0, st>>>(d_loge, d_loge_stats, prm, lt);
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch(4);
    // 4. backtrack over the whole sequence from the final chunk's argmax
    lay1.last = lay.last + (C - 1);
    return run_backtrack(lay1, hp1, 1, out_stride, d_states, st);
}

extern "C" int64_t iss_viterbi_work_bytes(int64_t total_steps, int n_seg)
{
    if (total_steps < 0 || n_seg < 0) return -1;
    const int64_t nc = total_steps / CH + n_seg + 1;
    const int64_t chunked = (total_steps / ECH + 2) * 256 + 8192;         // tables of the chunk-parallel energy pass
    return total_steps + 2 * nc + 3 * (int64_t)sizeof(int64_t) * (n_seg + 1) + n_seg + 9 * 256 + 1024 /* vin/vout/map scratch */ + chunked;
}

// One serial chain per recording: recording r is loge[h_off[r] .. h_off[r+1]) with statistics stats[2r ..] (stats_stride
// 2) or the one shared pair (stats_stride 0); every out_stride-th state goes to d_states[h_out_off[r] ..], or to
// d_states[0 ..] for a single recording (h_out_off == nullptr).
static int energy_chains(iss_ctx *ctx, const float *d_loge, const int64_t *h_off, int n_rec, const double *d_loge_stats,
                         int stats_stride, const VitParams &prm, int out_stride, const int64_t *h_out_off, uint8_t *d_states,
                         void *d_work, cudaStream_t st)
{
    HostPlan hp; VitLayout lay = {};
    int rc = make_layout(h_off, n_rec, d_work, hp, lay, st);
    if (rc != ISS_OK) return rc;
    lay.store_bp = 1;
    lay.stats_stride = stats_stride;
    if (h_out_off) {
        int64_t *d_out_off = reinterpret_cast<int64_t *>(lay.last + align_up((size_t)n_rec, 256));
        ISS_CUDA_OK(cudaMemcpyAsync(d_out_off, h_out_off, sizeof(int64_t) * n_rec, cudaMemcpyHostToDevice, st));
        lay.out_off = d_out_off;
    }
    viterbi_forward_kernel<2, true><<<n_rec, 32, 0, st>>>(d_loge, d_loge_stats, prm, lay);
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch();
    return run_backtrack(lay, hp, n_rec, out_stride, d_states, st);
}

extern "C" int iss_energy_viterbi(iss_ctx *ctx, const float *d_loge, int64_t L, const double *d_loge_stats,
                                  double log_ratio, const double *h_emis, const double *h_trans,
                                  double log_prior, int out_stride, uint8_t *d_states, void *d_work,
                                  void *stream)
{
    ISS_REQUIRE(ctx && h_emis && h_trans, ISS_ERR_INVALID, "iss_energy_viterbi: NULL argument");
    ISS_REQUIRE(out_stride >= 1, ISS_ERR_INVALID, "iss_energy_viterbi: out_stride must be >= 1");
    if (L <= 0) return ISS_OK;
    ISS_REQUIRE(d_loge && d_loge_stats && d_states && d_work, ISS_ERR_INVALID, "iss_energy_viterbi: NULL buffer");
    ISS_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = iss_stream(stream);
    VitParams prm = {};
    fill_energy_params(prm, h_emis, h_trans, log_prior, log_ratio);
    if (!energy_serial() && L >= 4 * ECH) return energy_viterbi_chunked(ctx, d_loge, L, d_loge_stats, prm, out_stride, d_states, d_work, st);
    const int64_t off[2] = {0, L};
    return energy_chains(ctx, d_loge, off, 1, d_loge_stats, 0, prm, out_stride, nullptr, d_states, d_work, st);
}

extern "C" int iss_energy_viterbi_multi(iss_ctx *ctx, const float *d_loge, const int64_t *h_loge_off, int n_rec,
                                        const double *d_loge_stats, double log_ratio, const double *h_emis,
                                        const double *h_trans, double log_prior, int out_stride,
                                        const int64_t *h_out_off, uint8_t *d_states, void *d_work, void *stream)
{
    ISS_REQUIRE(ctx && h_emis && h_trans && h_loge_off && h_out_off && n_rec >= 1, ISS_ERR_INVALID, "iss_energy_viterbi_multi: bad argument");
    ISS_REQUIRE(out_stride >= 1, ISS_ERR_INVALID, "iss_energy_viterbi_multi: out_stride must be >= 1");
    for (int r = 0; r < n_rec; ++r) {
        const int64_t L = h_loge_off[r + 1] - h_loge_off[r];
        ISS_REQUIRE(L >= 0 && L < 4 * ECH, ISS_ERR_INVALID,
                    "iss_energy_viterbi_multi: recording %d has %lld frames (>= %lld are decoded by iss_energy_viterbi)",
                    r, (long long)L, (long long)(4 * ECH));
    }
    if (h_loge_off[n_rec] == h_loge_off[0]) return ISS_OK;
    ISS_REQUIRE(d_loge && d_loge_stats && d_states && d_work, ISS_ERR_INVALID, "iss_energy_viterbi_multi: NULL buffer");
    ISS_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = iss_stream(stream);
    VitParams prm = {};
    fill_energy_params(prm, h_emis, h_trans, log_prior, log_ratio);
    return energy_chains(ctx, d_loge, h_loge_off, n_rec, d_loge_stats, 2, prm, out_stride, h_out_off, d_states, d_work, st);
}

extern "C" int iss_viterbi_segments(iss_ctx *ctx, const float *d_probs, int K, const int64_t *h_seg_off,
                                    int n_seg, const double *h_trans, double log_prior, uint8_t *d_states,
                                    void *d_work, void *stream)
{
    ISS_REQUIRE(ctx && h_seg_off && h_trans, ISS_ERR_INVALID, "iss_viterbi_segments: NULL argument");
    ISS_REQUIRE(K >= 2 && K <= MAXK, ISS_ERR_UNSUPPORTED, "iss_viterbi_segments: K=%d not in [2,4]", K);
    if (n_seg <= 0 || h_seg_off[n_seg] == 0) return ISS_OK;
    ISS_REQUIRE(d_probs && d_states && d_work, ISS_ERR_INVALID, "iss_viterbi_segments: NULL buffer");
    ISS_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = iss_stream(stream);
    HostPlan hp; VitLayout lay = {};
    int rc = make_layout(h_seg_off, n_seg, d_work, hp, lay, st);
    if (rc != ISS_OK) return rc;
    lay.store_bp = 1;
    VitParams prm = {};
    for (int i = 0; i < K; ++i) for (int j = 0; j < K; ++j) prm.A[i][j] = h_trans[i * K + j];
    prm.prior = log_prior;
    // shift the views so that segment offsets index d_probs rows directly
    if (K == 2) viterbi_forward_kernel<2, false><<<n_seg, 32, 0, st>>>(d_probs, nullptr, prm, lay);
    else if (K == 3) viterbi_forward_kernel<3, false><<<n_seg, 32, 0, st>>>(d_probs, nullptr, prm, lay);
    else viterbi_forward_kernel<4, false><<<n_seg, 32, 0, st>>>(d_probs, nullptr, prm, lay);
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch();
    return run_backtrack(lay, hp, n_seg, 1, d_states, st);
}

// ---- online decoding of live streams (stream.py) ----------------------------------------------------------------
// Many chains, each continued by one call from its carried scores.  A chain's undecided steps keep their back-pointer
// bytes in its history row.  After the forward steps the chain's K end states are traced back together: the latest step
// at which all K paths meet is the merge point m, and every state up to m is final.  Every path that ends optimally
// later passes through one of the K states traced back from, and their back-pointers never change, so the decided
// states are exactly those of the offline decode of the whole chain.  A chain flagged as ending is traced back in full
// from the first argmax, as the offline backtrack does.
namespace {

struct OnlineChain {
    int64_t src;                   // first step in d_src (energy: loge entry; CNN: posterior row)
    int64_t n;                     // new steps
    int64_t slot;                  // row of the scores / history / threshold tables
    int64_t pend;                  // undecided steps already in the history row
    int64_t out;                   // first decided state in d_out
    int64_t flags;                 // ISS_ONLINE_START | ISS_ONLINE_END
};

template <int K, bool ENERGY>
__global__ void __launch_bounds__(32)
viterbi_online_kernel(const float *__restrict__ src, const double *__restrict__ stats, VitParams prm,
                      const OnlineChain *__restrict__ chains, double *__restrict__ scores, uint8_t *__restrict__ hist,
                      int64_t hist_cap, uint8_t *__restrict__ out, int64_t *__restrict__ ndec)
{
    const OnlineChain c = chains[blockIdx.x];
    const int lane = threadIdx.x;
    const bool start = (c.flags & 1) != 0, end = (c.flags & 2) != 0;
    uint8_t *h = hist + c.slot * hist_cap;
    const double thr = ENERGY ? energy_threshold(stats + 2 * c.slot, prm.log_ratio) : 0.0;
    double V[K];
#pragma unroll
    for (int j = 0; j < K; ++j) V[j] = start ? 0.0 : scores[c.slot * MAXK + j];

    for (int64_t base = 0; base < c.n; base += 32) {
        const int64_t t = base + lane;
        double e[K];
#pragma unroll
        for (int j = 0; j < K; ++j) e[j] = 0.0;
        if (t < c.n) load_emissions<K, ENERGY>(src, c.src + t, thr, prm, e);
        const int nstep = (int)min((int64_t)32, c.n - base);
        unsigned mybp = 0;
        for (int s = 0; s < nstep; ++s) {
            double es[K];
#pragma unroll
            for (int j = 0; j < K; ++j) es[j] = __shfl_sync(0xffffffffu, e[j], s);
            const unsigned bp = vit_step<K, ENERGY>(V, es, prm, start && base + s == 0);
            if (lane == s) mybp = bp;
        }
        if (t < c.n) h[c.pend + t] = (uint8_t)mybp;
    }
    __syncwarp();                                      // the lanes' back-pointer stores are visible to lane 0

    const int64_t P = c.pend + c.n;                    // undecided steps: h[0 .. P)
    int64_t nd = 0;
    if (lane == 0) {
        int64_t m = -1;                                // last decided step
        unsigned x = 0;
        if (end) {
            m = P - 1;
            x = (unsigned)first_argmax<K>(V);
        } else {
            unsigned map = 0xE4;                       // end state -> state at step i (identity at i = P - 1)
            for (int64_t i = P - 1; i >= 0; --i) {
                bool same = true;
#pragma unroll
                for (int k = 1; k < K; ++k) same = same && (((map >> (2 * k)) & 3) == (map & 3));
                if (same) { m = i; x = map & 3; break; }
                if (i == 0) break;
                map = compose_map(h[i], map);
            }
        }
        for (int64_t r = m; r >= 0; --r) {
            out[c.out + r] = (uint8_t)x;
            if (r > 0) x = (h[r] >> (2 * x)) & 3;
        }
        nd = m + 1;
        ndec[blockIdx.x] = nd;
#pragma unroll
        for (int k = 0; k < K; ++k) scores[c.slot * MAXK + k] = V[k];
    }
    nd = __shfl_sync(0xffffffffu, nd, 0);
    if (end || nd == 0) return;
    // drop the decided steps: h[nd .. P) -> h[0 .. P - nd), 32 bytes per round, reads before writes
    for (int64_t b = 0; b < P - nd; b += 32) {
        const int64_t i = b + lane;
        const uint8_t v = i < P - nd ? h[nd + i] : 0;
        __syncwarp();
        if (i < P - nd) h[i] = v;
        __syncwarp();
    }
}

template <int K, bool ENERGY>
void launch_online(int n, cudaStream_t st, const float *src, const double *stats, const VitParams &prm,
                   const OnlineChain *chains, double *scores, uint8_t *hist, int64_t hist_cap, uint8_t *out, int64_t *ndec)
{
    viterbi_online_kernel<K, ENERGY><<<n, 32, 0, st>>>(src, stats, prm, chains, scores, hist, hist_cap, out, ndec);
}

}  // namespace

extern "C" int64_t iss_viterbi_online_work_bytes(int n_chain)
{
    return n_chain < 0 ? -1 : (int64_t)sizeof(OnlineChain) * n_chain;
}

extern "C" int iss_viterbi_online(iss_ctx *ctx, int K, int n_chain, const int64_t *h_chains, const float *d_src,
                                  int64_t src_len, const double *d_stats, double log_ratio, const double *h_emis,
                                  const double *h_trans, double log_prior, double *d_scores, uint8_t *d_hist,
                                  int64_t n_slots, int64_t hist_cap, uint8_t *d_out, int64_t out_len, int64_t *d_ndec,
                                  void *d_work, void *stream)
{
    const bool energy = h_emis != nullptr;
    ISS_REQUIRE(ctx && h_trans && n_chain >= 0, ISS_ERR_INVALID, "iss_viterbi_online: bad argument");
    ISS_REQUIRE(K >= 2 && K <= MAXK && (!energy || K == 2), ISS_ERR_UNSUPPORTED, "iss_viterbi_online: K=%d not supported", K);
    if (n_chain == 0) return ISS_OK;
    ISS_REQUIRE(h_chains && d_scores && d_hist && d_out && d_ndec && d_work && (!energy || d_stats), ISS_ERR_INVALID,
                "iss_viterbi_online: NULL buffer");
    for (int i = 0; i < n_chain; ++i) {
        const int64_t *c = h_chains + 6 * i;
        ISS_REQUIRE(c[1] >= 0 && c[2] >= 0 && c[3] >= 0 && c[4] >= 0 && (c[1] == 0 || c[0] >= 0), ISS_ERR_INVALID,
                    "iss_viterbi_online: chain %d: negative field", i);
        ISS_REQUIRE(c[1] == 0 || c[0] + c[1] <= src_len, ISS_ERR_INVALID,
                    "iss_viterbi_online: chain %d: steps %lld .. %lld outside d_src (%lld steps)", i, (long long)c[0],
                    (long long)(c[0] + c[1]), (long long)src_len);
        ISS_REQUIRE(c[2] < n_slots, ISS_ERR_INVALID, "iss_viterbi_online: chain %d: slot %lld of %lld", i,
                    (long long)c[2], (long long)n_slots);
        ISS_REQUIRE(c[4] + c[3] + c[1] <= out_len, ISS_ERR_INVALID,
                    "iss_viterbi_online: chain %d: decided states %lld .. %lld outside d_out (%lld)", i, (long long)c[4],
                    (long long)(c[4] + c[3] + c[1]), (long long)out_len);
        ISS_REQUIRE(c[3] + c[1] <= hist_cap, ISS_ERR_INVALID,
                    "iss_viterbi_online: chain %d: %lld undecided steps exceed the history capacity %lld", i,
                    (long long)(c[3] + c[1]), (long long)hist_cap);
        ISS_REQUIRE(!(c[5] & 1) || (c[3] == 0 && c[1] > 0), ISS_ERR_INVALID,
                    "iss_viterbi_online: chain %d starts without steps or with a history", i);
        ISS_REQUIRE(c[1] == 0 || d_src, ISS_ERR_INVALID, "iss_viterbi_online: NULL d_src");
    }
    ISS_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = iss_stream(stream);
    OnlineChain *d_chains = reinterpret_cast<OnlineChain *>(d_work);
    ISS_CUDA_OK(cudaMemcpyAsync(d_chains, h_chains, sizeof(OnlineChain) * n_chain, cudaMemcpyHostToDevice, st));
    VitParams prm = {};
    if (energy) fill_energy_params(prm, h_emis, h_trans, log_prior, log_ratio);
    else {
        for (int i = 0; i < K; ++i) for (int j = 0; j < K; ++j) prm.A[i][j] = h_trans[i * K + j];
        prm.prior = log_prior;
    }
    if (energy) launch_online<2, true>(n_chain, st, d_src, d_stats, prm, d_chains, d_scores, d_hist, hist_cap, d_out, d_ndec);
    else if (K == 2) launch_online<2, false>(n_chain, st, d_src, nullptr, prm, d_chains, d_scores, d_hist, hist_cap, d_out, d_ndec);
    else if (K == 3) launch_online<3, false>(n_chain, st, d_src, nullptr, prm, d_chains, d_scores, d_hist, hist_cap, d_out, d_ndec);
    else launch_online<4, false>(n_chain, st, d_src, nullptr, prm, d_chains, d_scores, d_hist, hist_cap, d_out, d_ndec);
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch();
    return ISS_OK;
}
