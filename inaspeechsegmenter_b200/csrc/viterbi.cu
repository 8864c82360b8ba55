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
// chain: the 32 lanes fetch and convert 32 steps of emissions in parallel
// (coalesced), then replay them through register shuffles while every lane
// carries the same V; lane j keeps step j's back-pointer byte so stores are
// coalesced too (forward_steps).  The backtrack -- pure integer function
// composition, hence associative and exact -- is parallel: per-256-step chunk
// maps, a short serial scan over chunk maps, then all chunks emit their states
// concurrently.
//
// Structure: an offline entry point carves its workspace with carve(), whose
// layout depends only on the sizes of the decode, names the chains of each
// forward launch with a VitChains (which sequence a block walks, where its
// scores come from and go to, where its argmax and back-pointers go), and
// backtracks with run_backtrack.  The online kernel for live streams runs the
// same forward_steps and traces back its own history rows.
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <type_traits>
#include <vector>

#include "iss_common.cuh"

namespace {

constexpr int CH = 256;            // backtrack chunk (steps)
constexpr int MAXK = 4;
constexpr int64_t ECH = 16384;     // chunk of the chunk-parallel energy decode (steps)

struct VitParams {
    double A[MAXK][MAXK];          // from -> to
    double prior;
    double emis_hit, emis_miss;    // energy mode
    double log_ratio;
};

// energy mode (K = 2) when h_emis is given, CNN posteriors otherwise
VitParams make_params(int K, const double *h_trans, double log_prior, const double *h_emis, double log_ratio)
{
    VitParams prm = {};
    for (int i = 0; i < K; ++i) for (int j = 0; j < K; ++j) prm.A[i][j] = h_trans[i * K + j];
    prm.prior = log_prior;
    if (h_emis) { prm.emis_hit = h_emis[0]; prm.emis_miss = h_emis[1]; prm.log_ratio = log_ratio; }
    return prm;
}

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// The regions of d_work.  A chain is one warp's forward walk over one sequence, or over one ECH chunk of it.
struct VitWork {
    uint8_t *bp;                   // [total] one byte per step: 2 bits per destination state
    uint8_t *cmap;                 // [chunks] composite back map of each backtrack chunk
    uint8_t *cend;                 // [chunks] state at the last step of each backtrack chunk
    int64_t *seq_off;              // [n_seq + 1] steps of each sequence
    int64_t *chunk_off;            // [n_seq + 1] backtrack chunks of each sequence
    int64_t *out_off;              // [n_seq] first output of each sequence (several recordings)
    uint8_t *last;                 // [chains] first argmax of each chain's final scores
    double *vin;                   // [chains][MAXK] incoming scores of each chain
    double *vout;                  // [chains][MAXK] outgoing scores V[T-1] of each chain
    uint8_t *map;                  // [1] composite back map of the whole of sequence 0
    int64_t *ech_off;              // [n_ech + 1] chunk-parallel energy decode: steps of each ECH chunk
    double *entry;                 // [n_ech][MAXK] scores entering each ECH chunk
    size_t bytes;
};

// The one layout of d_work for a decode of `total` steps in n_seq sequences, a function of the sizes only: so
// iss_energy_forward and iss_energy_emit find the same tables in the d_work they share, and iss_viterbi_work_bytes
// is the layout on a null base.
VitWork carve(void *base, int64_t total, int n_seq)
{
    const int64_t chunks = total / CH + n_seq;                          // >= the chunks of any n_seq sequences
    const int64_t n_ech = (total + ECH - 1) / ECH;
    const int64_t chains = std::max<int64_t>(n_seq, 2 * n_ech);         // one per sequence or two per ECH chunk
    VitWork w;
    size_t o = 0;
    auto take = [&](auto *&p, int64_t n) {
        p = reinterpret_cast<std::remove_reference_t<decltype(p)>>(reinterpret_cast<uintptr_t>(base) + o);
        o = align_up(o + sizeof(*p) * (size_t)n, 256);
    };
    take(w.bp, total);
    take(w.cmap, chunks);
    take(w.cend, chunks);
    take(w.seq_off, n_seq + 1);
    take(w.chunk_off, n_seq + 1);
    take(w.out_off, n_seq);
    take(w.last, chains);
    take(w.vin, chains * MAXK);
    take(w.vout, chains * MAXK);
    take(w.map, 1);
    take(w.ech_off, n_ech + 1);
    take(w.entry, n_ech * MAXK);
    w.bytes = o;
    return w;
}

// The chains of one forward launch: block b walks sequence s = first + b / per_seq of seq_off as chain
// c = first * per_seq + b (per_seq = 2: the two basis chains of a transfer matrix).  Chain c starts from the scores
// vin[c], or from the prior on the sequence's first step when vin is null; it leaves its final scores in vout[c] and
// their first argmax in last[c], and its back-pointers at the sequence's steps of bp, where those are not null.
// Energy mode thresholds sequence s on stats[s * stats_stride ..].
struct VitChains {
    const int64_t *seq_off;
    int first, per_seq;
    const double *vin;
    double *vout;
    uint8_t *last;
    uint8_t *bp;
    int stats_stride;
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
        for (int j = 0; j < K; ++j)                     // float32(log(double p)): a correctly rounded float32 log.
            e[j] = (double)(float)log((double)src[i * K + j]);   // numpy's float32 log is not (DESIGN, "Emission log")
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

// Steps [0, T) of one chain whose emissions start at step s0 of src, with every lane carrying the same V.  `first`:
// step 0 is the first step of the sequence (the prior).  Lane i of each round of 32 steps hands the back-pointer
// byte of step t = base + i to store(t, byte).
template <int K, bool ENERGY, typename Store>
__device__ __forceinline__ void forward_steps(const float *__restrict__ src, int64_t s0, int64_t T, double thr,
                                              const VitParams &prm, bool first, double (&V)[K], Store store)
{
    const int lane = threadIdx.x;
    for (int64_t base = 0; base < T; base += 32) {
        const int64_t t = base + lane;
        double e[K];
#pragma unroll
        for (int j = 0; j < K; ++j) e[j] = 0.0;
        if (t < T) load_emissions<K, ENERGY>(src, s0 + t, thr, prm, e);
        const int nstep = (int)min((int64_t)32, T - base);
        unsigned mybp = 0;
        if (nstep == 32 && (base > 0 || !first)) {
            // full block, fully unrolled: the 32 x K emission shuffles do not depend on V, so they are
            // issued ahead and only the add/compare/select chain remains on the serial critical path
#pragma unroll
            for (int s = 0; s < 32; ++s) {
                double es[K];
#pragma unroll
                for (int j = 0; j < K; ++j) es[j] = __shfl_sync(0xffffffffu, e[j], s);
                const unsigned bp = vit_step<K, ENERGY>(V, es, prm, false);
                mybp = (lane == s) ? bp : mybp;
            }
        } else {
            for (int s = 0; s < nstep; ++s) {
                double es[K];
#pragma unroll
                for (int j = 0; j < K; ++j) es[j] = __shfl_sync(0xffffffffu, e[j], s);
                const unsigned bp = vit_step<K, ENERGY>(V, es, prm, first && base + s == 0);
                if (lane == s) mybp = bp;
            }
        }
        if (t < T) store(t, mybp);
    }
}

template <int K, bool ENERGY>
__global__ void __launch_bounds__(32)
viterbi_forward_kernel(const float *__restrict__ src, const double *__restrict__ stats, VitParams prm, VitChains ch)
{
    const int c = ch.first * ch.per_seq + blockIdx.x, s = c / ch.per_seq;
    const int64_t t0 = ch.seq_off[s];
    const int64_t T = ch.seq_off[s + 1] - t0;
    if (T <= 0) return;
    const bool cont = ch.vin != nullptr;           // first step is an ordinary transition from vin
    const double thr = ENERGY ? energy_threshold(stats + (int64_t)s * ch.stats_stride, prm.log_ratio) : 0.0;
    double V[K];
#pragma unroll
    for (int j = 0; j < K; ++j) V[j] = cont ? ch.vin[c * MAXK + j] : 0.0;
    forward_steps<K, ENERGY>(src, t0, T, thr, prm, !cont, V, [&](int64_t t, unsigned b) {
        if (ch.bp) ch.bp[t0 + t] = (uint8_t)b;
    });
    if (threadIdx.x == 0) {
        if (ch.last) ch.last[c] = (uint8_t)first_argmax<K>(V);
        if (ch.vout) {
#pragma unroll
            for (int k = 0; k < K; ++k) ch.vout[c * MAXK + k] = V[k];
        }
    }
}

__device__ __forceinline__ int find_seg(const int64_t *chunk_off, int n_seq, int64_t c)
{
    int lo = 0, hi = n_seq;            // chunk_off[lo] <= c < chunk_off[hi]
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (chunk_off[mid] <= c) lo = mid; else hi = mid;
    }
    return lo;
}

// cmap[c]: (state at the last step of chunk c) -> (state at the last step of chunk c-1)
__global__ void viterbi_chunk_map_kernel(VitWork w, int n_seq, int64_t nchunks, int has_pred)
{
    const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nchunks) return;
    const int seg = find_seg(w.chunk_off, n_seq, c);
    const int64_t t0 = w.seq_off[seg], T = w.seq_off[seg + 1] - t0;
    const int64_t lc = c - w.chunk_off[seg];
    const int64_t a = lc * CH, b = min(a + CH, T);          // steps [a, b)
    unsigned m = 0xE4;                                      // identity: 3,2,1,0 in 2-bit fields
    const uint8_t *bp = w.bp + t0;
    for (int64_t t = b - 1; t >= a; --t) {
        if (t == 0 && !has_pred) break;                     // bp[0] is unused when the sequence has no predecessor
        m = compose_map(bp[t], m);
    }
    w.cmap[c] = (uint8_t)m;
}

// serial over the chunks of one sequence (T/256 steps), one thread per sequence, which starts from the argmax of
// chain end_chain + seg (the chain that walked its last step)
__global__ void viterbi_chunk_scan_kernel(VitWork w, int n_seq, int end_chain)
{
    const int seg = blockIdx.x * blockDim.x + threadIdx.x;
    if (seg >= n_seq) return;
    const int64_t c0 = w.chunk_off[seg], c1 = w.chunk_off[seg + 1];
    if (c1 <= c0) return;
    unsigned x = w.last[end_chain + seg];
    for (int64_t c = c1 - 1; c >= c0; --c) {
        w.cend[c] = (uint8_t)x;
        x = (w.cmap[c] >> (2 * x)) & 3;
    }
}

// every out_stride-th state of sequence seg to states[out_off[seg] ..], or to states[seq_off[seg] ..] when out_off is
// null (a single sequence has seq_off[0] == 0)
__global__ void viterbi_chunk_emit_kernel(VitWork w, int n_seq, int64_t nchunks, const int64_t *__restrict__ out_off,
                                          int out_stride, uint8_t *__restrict__ states)
{
    const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nchunks) return;
    const int seg = find_seg(w.chunk_off, n_seq, c);
    const int64_t t0 = w.seq_off[seg], T = w.seq_off[seg + 1] - t0;
    const int64_t lc = c - w.chunk_off[seg];
    const int64_t a = lc * CH, b = min(a + CH, T);
    const uint8_t *bp = w.bp + t0;
    unsigned x = w.cend[c];
    const int64_t o0 = out_off ? out_off[seg] : t0;
    for (int64_t t = b - 1; t >= a; --t) {
        if (out_stride == 1) states[o0 + t] = (uint8_t)x;
        else if (t % out_stride == 0) states[o0 + t / out_stride] = (uint8_t)x;
        x = (bp[t] >> (2 * x)) & 3;
    }
}

// composite of all chunk maps of sequence 0: (state at the last step) -> (state just before the first step)
__global__ void viterbi_compose_kernel(VitWork w, int64_t nchunks)
{
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    unsigned m = 0xE4;
    for (int64_t c = nchunks - 1; c >= 0; --c) m = compose_map(w.cmap[c], m);
    w.map[0] = (uint8_t)m;
}

// Uploads the offsets of n_seq sequences and of their backtrack chunks; *nchunks = the number of chunks.
int upload_offsets(const VitWork &w, const int64_t *h_seq_off, int n_seq, int64_t *nchunks, cudaStream_t st)
{
    std::vector<int64_t> seq_off(h_seq_off, h_seq_off + n_seq + 1), chunk_off(n_seq + 1);
    int64_t nc = 0;
    for (int s = 0; s < n_seq; ++s) {
        chunk_off[s] = nc;
        const int64_t T = seq_off[s + 1] - seq_off[s];
        ISS_REQUIRE(T >= 0, ISS_ERR_INVALID, "viterbi: segment offsets must be non-decreasing");
        nc += (T + CH - 1) / CH;
    }
    chunk_off[n_seq] = nc;
    *nchunks = nc;
    ISS_CUDA_OK(cudaMemcpyAsync(w.seq_off, seq_off.data(), sizeof(int64_t) * (n_seq + 1), cudaMemcpyHostToDevice, st));
    ISS_CUDA_OK(cudaMemcpyAsync(w.chunk_off, chunk_off.data(), sizeof(int64_t) * (n_seq + 1), cudaMemcpyHostToDevice, st));
    return ISS_OK;
}

int run_backtrack(const VitWork &w, int n_seq, int64_t nchunks, int end_chain, const int64_t *out_off, int out_stride,
                  uint8_t *d_states, cudaStream_t st)
{
    if (nchunks == 0) return ISS_OK;
    const int TB = 128;
    const unsigned gc = (unsigned)((nchunks + TB - 1) / TB);
    viterbi_chunk_map_kernel<<<gc, TB, 0, st>>>(w, n_seq, nchunks, 0);
    viterbi_chunk_scan_kernel<<<(n_seq + 63) / 64, 64, 0, st>>>(w, n_seq, end_chain);
    viterbi_chunk_emit_kernel<<<gc, TB, 0, st>>>(w, n_seq, nchunks, out_off, out_stride, d_states);
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch(3);
    return ISS_OK;
}

// One chain per sequence h_off[s] .. h_off[s+1] of src, then the backtrack: every out_stride-th state of sequence s
// goes to d_states[h_out_off[s] ..], or to d_states[h_off[s] ..] when h_out_off is null.
template <int K, bool ENERGY>
int decode_sequences(const float *src, const int64_t *h_off, int n_seq, const double *stats, int stats_stride,
                     const VitParams &prm, int out_stride, const int64_t *h_out_off, uint8_t *d_states, void *d_work,
                     cudaStream_t st)
{
    const VitWork w = carve(d_work, h_off[n_seq], n_seq);
    int64_t nc;
    int rc = upload_offsets(w, h_off, n_seq, &nc, st);
    if (rc != ISS_OK) return rc;
    if (h_out_off) ISS_CUDA_OK(cudaMemcpyAsync(w.out_off, h_out_off, sizeof(int64_t) * n_seq, cudaMemcpyHostToDevice, st));
    const VitChains ch = {w.seq_off, 0, 1, nullptr, nullptr, w.last, w.bp, stats_stride};
    viterbi_forward_kernel<K, ENERGY><<<n_seq, 32, 0, st>>>(src, stats, prm, ch);
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch();
    return run_backtrack(w, n_seq, nc, 0, h_out_off ? w.out_off : nullptr, out_stride, d_states, st);
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
// (ISS_B200_VITERBI=serial); the GPU tests compare both with the C oracle, 10 h tracks included.
//
// Chain c is chunk c in steps 1a and 3; chains 2c and 2c + 1 are the basis chains of chunk c in step 1b.
__global__ void energy_entry_compose_kernel(VitWork w, int n_ech)
{
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    double e0 = w.vout[0], e1 = w.vout[1];                       // scores leaving chunk 0 = entering chunk 1
    for (int c = 1; c < n_ech; ++c) {
        w.entry[c * MAXK + 0] = e0; w.entry[c * MAXK + 1] = e1;
        // vout of chain 2c + i = scores leaving chunk c when entering in state i with score 0
        const double *m0 = w.vout + (size_t)(2 * c) * MAXK, *m1 = m0 + MAXK;
        const double a0 = e0 + m0[0], b0 = e1 + m1[0], a1 = e0 + m0[1], b1 = e1 + m1[1];
        e0 = (b0 > a0) ? b0 : a0;
        e1 = (b1 > a1) ? b1 : a1;
    }
}

int energy_viterbi_chunked(const float *d_loge, int64_t L, const double *d_loge_stats, const VitParams &prm,
                           int out_stride, uint8_t *d_states, void *d_work, cudaStream_t st)
{
    const int C = (int)((L + ECH - 1) / ECH);
    const VitWork w = carve(d_work, L, 1);
    const int64_t off[2] = {0, L};                               // the backtrack: ONE sequence [0, L)
    int64_t nc;
    int rc = upload_offsets(w, off, 1, &nc, st);
    if (rc != ISS_OK) return rc;
    std::vector<int64_t> ech_off(C + 1);
    for (int c = 0; c <= C; ++c) ech_off[c] = std::min<int64_t>((int64_t)c * ECH, L);
    ISS_CUDA_OK(cudaMemcpyAsync(w.ech_off, ech_off.data(), sizeof(int64_t) * (C + 1), cudaMemcpyHostToDevice, st));
    std::vector<double> basis((size_t)MAXK * 2 * C, 0.0);
    for (int c = 0; c < C; ++c) {                                // e_0 = (0, -inf), e_1 = (-inf, 0) in max-plus
        basis[(size_t)(2 * c) * MAXK + 1] = -INFINITY;
        basis[(size_t)(2 * c + 1) * MAXK + 0] = -INFINITY;
    }
    ISS_CUDA_OK(cudaMemcpyAsync(w.vin, basis.data(), sizeof(double) * basis.size(), cudaMemcpyHostToDevice, st));
    // 1a. chunk 0, true pass (prior on the first frame), back-pointers stored
    const VitChains c0 = {w.ech_off, 0, 1, nullptr, w.vout, nullptr, w.bp, 0};
    viterbi_forward_kernel<2, true><<<1, 32, 0, st>>>(d_loge, d_loge_stats, prm, c0);
    // 1b. chunks 1..C-1: two basis chains each
    const VitChains cb = {w.ech_off, 1, 2, w.vin, w.vout, nullptr, nullptr, 0};
    viterbi_forward_kernel<2, true><<<2 * (C - 1), 32, 0, st>>>(d_loge, d_loge_stats, prm, cb);
    // 2. entry scores of chunks 1..C-1
    energy_entry_compose_kernel<<<1, 32, 0, st>>>(w, C);
    // 3. chunks 1..C-1, true pass from their entry scores
    const VitChains ct = {w.ech_off, 1, 1, w.entry, nullptr, w.last, w.bp, 0};
    viterbi_forward_kernel<2, true><<<C - 1, 32, 0, st>>>(d_loge, d_loge_stats, prm, ct);
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch(4);
    // 4. backtrack over the whole sequence from the argmax of the last chunk's chain
    return run_backtrack(w, 1, nc, C - 1, nullptr, out_stride, d_states, st);
}

}  // namespace

extern "C" int64_t iss_viterbi_work_bytes(int64_t total_steps, int n_seg)
{
    if (total_steps < 0 || n_seg < 0) return -1;
    return (int64_t)carve(nullptr, total_steps, n_seg).bytes;
}

// ---- partial chains of the energy Viterbi for time-sharded recordings (SURVEY 8(e)) -------------------
extern "C" int iss_energy_transfer(iss_ctx *ctx, const float *d_loge, int64_t L, const double *d_loge_stats,
                                   double log_ratio, const double *h_emis, const double *h_trans,
                                   double *h_matrix, void *d_work, void *stream)
{
    ISS_REQUIRE(ctx && d_loge && d_loge_stats && h_emis && h_trans && h_matrix && d_work && L > 0, ISS_ERR_INVALID, "iss_energy_transfer: bad argument");
    ISS_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = iss_stream(stream);
    const VitWork w = carve(d_work, L, 1);
    const int64_t off[2] = {0, L};
    int64_t nc;
    int rc = upload_offsets(w, off, 1, &nc, st);
    if (rc != ISS_OK) return rc;
    const double NEG_INF = -INFINITY;
    double vin[2 * MAXK] = {0.0, NEG_INF, 0, 0, NEG_INF, 0.0, 0, 0};      // basis vectors e_0, e_1 (max-plus)
    ISS_CUDA_OK(cudaMemcpyAsync(w.vin, vin, sizeof(vin), cudaMemcpyHostToDevice, st));
    const VitChains ch = {w.seq_off, 0, 2, w.vin, w.vout, nullptr, nullptr, 0};
    viterbi_forward_kernel<2, true><<<2, 32, 0, st>>>(d_loge, d_loge_stats, make_params(2, h_trans, 0.0, h_emis, log_ratio), ch);
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch();
    double vout[2 * MAXK];
    ISS_CUDA_OK(cudaMemcpyAsync(vout, w.vout, sizeof(vout), cudaMemcpyDeviceToHost, st));
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
    const VitWork w = carve(d_work, L, 1);
    const int64_t off[2] = {0, L};
    int64_t nc;
    int rc = upload_offsets(w, off, 1, &nc, st);
    if (rc != ISS_OK) return rc;
    if (h_vin) {
        double vin[MAXK] = {h_vin[0], h_vin[1], 0, 0};
        ISS_CUDA_OK(cudaMemcpyAsync(w.vin, vin, sizeof(vin), cudaMemcpyHostToDevice, st));
    }
    const VitChains ch = {w.seq_off, 0, 1, h_vin ? w.vin : nullptr, w.vout, w.last, w.bp, 0};
    viterbi_forward_kernel<2, true><<<1, 32, 0, st>>>(d_loge, d_loge_stats, make_params(2, h_trans, log_prior, h_emis, log_ratio), ch);
    const unsigned gc = (unsigned)((nc + 127) / 128);
    viterbi_chunk_map_kernel<<<gc, 128, 0, st>>>(w, 1, nc, h_vin ? 1 : 0);
    viterbi_compose_kernel<<<1, 32, 0, st>>>(w, nc);
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch(3);
    double vout[MAXK];
    uint8_t m;
    ISS_CUDA_OK(cudaMemcpyAsync(vout, w.vout, sizeof(vout), cudaMemcpyDeviceToHost, st));
    ISS_CUDA_OK(cudaMemcpyAsync(&m, w.map, 1, cudaMemcpyDeviceToHost, st));
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
    const VitWork w = carve(d_work, L, 1);                      // iss_energy_forward's tables, already on the device
    const int64_t nc = (L + CH - 1) / CH;
    if (end_state >= 0) ISS_CUDA_OK(cudaMemsetAsync(w.last, end_state, 1, st));
    viterbi_chunk_scan_kernel<<<1, 64, 0, st>>>(w, 1, 0);
    viterbi_chunk_emit_kernel<<<(unsigned)((nc + 127) / 128), 128, 0, st>>>(w, 1, nc, nullptr, out_stride, d_states);
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch(3);
    return ISS_OK;
}

// ---- whole recordings and CNN segments --------------------------------------------------------------------
static int g_energy_serial = -1;        // -1: read ISS_B200_VITERBI on first use
static bool energy_serial()
{
    if (g_energy_serial < 0) { const char *e = getenv("ISS_B200_VITERBI"); g_energy_serial = (e && !strcmp(e, "serial")) ? 1 : 0; }
    return g_energy_serial == 1;
}
extern "C" int iss_set_energy_viterbi_serial(int serial) { g_energy_serial = serial ? 1 : 0; return ISS_OK; }

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
    const VitParams prm = make_params(2, h_trans, log_prior, h_emis, log_ratio);
    if (!energy_serial() && L >= 4 * ECH) return energy_viterbi_chunked(d_loge, L, d_loge_stats, prm, out_stride, d_states, d_work, st);
    const int64_t off[2] = {0, L};
    return decode_sequences<2, true>(d_loge, off, 1, d_loge_stats, 0, prm, out_stride, nullptr, d_states, d_work, st);
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
    return decode_sequences<2, true>(d_loge, h_loge_off, n_rec, d_loge_stats, 2, make_params(2, h_trans, log_prior, h_emis, log_ratio),
                                     out_stride, h_out_off, d_states, d_work, st);
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
    const VitParams prm = make_params(K, h_trans, log_prior, nullptr, 0.0);
    auto decode = K == 2 ? decode_sequences<2, false> : K == 3 ? decode_sequences<3, false> : decode_sequences<4, false>;
    return decode(d_probs, h_seg_off, n_seg, nullptr, 0, prm, 1, nullptr, d_states, d_work, st);
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
    forward_steps<K, ENERGY>(src, c.src, c.n, thr, prm, start, V, [&](int64_t t, unsigned b) { h[c.pend + t] = (uint8_t)b; });
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
    const VitParams prm = make_params(K, h_trans, log_prior, h_emis, log_ratio);
    if (energy) launch_online<2, true>(n_chain, st, d_src, d_stats, prm, d_chains, d_scores, d_hist, hist_cap, d_out, d_ndec);
    else if (K == 2) launch_online<2, false>(n_chain, st, d_src, nullptr, prm, d_chains, d_scores, d_hist, hist_cap, d_out, d_ndec);
    else if (K == 3) launch_online<3, false>(n_chain, st, d_src, nullptr, prm, d_chains, d_scores, d_hist, hist_cap, d_out, d_ndec);
    else launch_online<4, false>(n_chain, st, d_src, nullptr, prm, d_chains, d_scores, d_hist, hist_cap, d_out, d_ndec);
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch();
    return ISS_OK;
}
