// cnn.cu -- K2: sliding-patch z-normalisation + CNN forward (generic Keras-style
// Sequential: Conv2D / MaxPooling2D / Dense with fused bias + BatchNorm affine +
// ReLU epilogues, softmax head, non-finite override).
//
// Reference semantics: _get_patches (inaSpeechSegmenter/segmenter.py:76-88),
// DnnSegmenter.__call__ (:135-179: band select :146-147, gather of `inlabel`
// segments :156-162, keras predict :163, r[~finite] = 0.5 :175).  The network
// itself lives only in keras_*_cnn.hdf5 (not in the reference tree), so layers
// arrive as iss_layer_desc records (Keras channels_last semantics).
//
// Data layout: activations are NHWC float32 ([patch][row=time][col=mel][chan]),
// i.e. the implicit-GEMM A operand has K = (kh, kw, cin) contiguous in cin, and
// Keras kernels [kh][kw][cin][cout] are the row-major B operand [K][N] verbatim.
// The 68 x nmel patches are NEVER materialised (the reference builds ~1 GB per
// audio-hour per network): the first conv layer gathers straight from the
// log-mel rows and applies (x - mean) / std of its patch on the fly.
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <type_traits>
#include <vector>

#include "conv_gemm.cuh"

namespace {

constexpr int PATCH_H = 68;            // frames per patch (segmenter.py:149)
constexpr int PATCH_HOP = 2;           // patch hop in frames (segmenter.py:149)
constexpr int PATCH_LFILL = PATCH_H / (2 * PATCH_HOP);     // 17 left replicas (segmenter.py:83)
// patches per layer-by-layer sweep: 8192 measured 6 % faster than 2048 (fewer partial waves of the persistent kernels);
// ISS_B200_CNN_BATCH: experiments; read once -- the workspace is sized with it
static int cnn_batch()
{
    static const int b = [] { const char *e = getenv("ISS_B200_CNN_BATCH"); const int v = e ? atoi(e) : 0; return v >= 64 && v <= 16384 ? v : 8192; }();
    return b;
}
#define CNN_BATCH cnn_batch()

struct Layer {
    iss_layer_desc d;
    int in_h, in_w, in_c;
    int out_h, out_w, out_c;
    TcWeights wt;
};

// floating-point operations of one patch through the layer
double layer_flops(const Layer &L)
{
    if (L.d.kind == ISS_LAYER_CONV2D) return 2.0 * L.out_h * L.out_w * (double)L.d.kh * L.d.kw * L.d.cin * L.d.cout;
    if (L.d.kind == ISS_LAYER_DENSE) return 2.0 * (double)L.d.cin * L.d.cout;
    return 0.0;
}

}  // namespace

struct iss_cnn {
    iss_ctx *ctx;
    std::vector<Layer> layers;
    float *d_blob;
    int64_t blob_len;
    int in_h, in_w;
    int n_classes;
    int64_t max_act;       // largest per-patch activation (floats) over all layer outputs
    double flops;
    double *d_first_S = nullptr;   // [cout of layer 0] float64 sums of the first layer's filter taps (FirstFuse)
    // live profiling of one layer (bench.py roofline)
    int prof_layer = -1;
    std::vector<cudaEvent_t> prof_ev;      // pairs: [2i] start, [2i+1] stop
    size_t prof_used = 0;
    double prof_flops = 0;
};

namespace {

// ------------------------------------------------------------------ patch bookkeeping
struct PatchArrays {
    int32_t *row0;         // first log-mel row of the patch
    float *mu, *sigma;     // float32 statistics (population std)
    uint8_t *finite;
};

// A range of padded patch indices [start, start + its length) of the recording whose rows begin at row `base` and which
// has U un-replicated windows.
struct PatchRange {
    int64_t base, U;
    int32_t start;
};

// first log-mel row of patch p of a range (patch_index_kernel and the host's copy of it)
__host__ __device__ __forceinline__ int64_t patch_row0(const PatchRange &r, int64_t p, int edge_left, int edge_right)
{
    int64_t j = p - (edge_left ? PATCH_LFILL : 0);              // un-replicated window index
    if (j < 0) j = 0;
    if (edge_right && j > r.U - 1) j = r.U - 1;
    return r.base + j * PATCH_HOP;
}

__global__ void patch_index_kernel(const PatchRange *__restrict__ ranges, const int64_t *__restrict__ seg_off,
                                   int n_seg, int64_t n, int edge_left, int edge_right, int32_t *__restrict__ row0)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int lo = 0, hi = n_seg;
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (seg_off[mid] <= i) lo = mid; else hi = mid; }
    const PatchRange r = ranges[lo];
    row0[i] = (int32_t)patch_row0(r, r.start + (i - seg_off[lo]), edge_left, edge_right);     // padded patch index
}

// one warp per patch: mean / population std over the 68 x w values (np.mean / np.std, segmenter.py:82)
__global__ void __launch_bounds__(256)
patch_stats_kernel(const float *__restrict__ mspec, int ld, int w, int64_t n, PatchArrays pa)
{
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (i >= n) return;
    const float *base = mspec + (int64_t)pa.row0[i] * ld;
    const int cnt = PATCH_H * w;
    double s1 = 0.0, s2 = 0.0;
    for (int e = lane; e < cnt; e += 32) {
        const int r = e / w, c = e - r * w;
        const double v = (double)base[r * ld + c];
        s1 += v; s2 += v * v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
    if (lane == 0) {
        const double m = s1 / cnt;
        double var = s2 / cnt - m * m;
        if (var < 0.0) var = 0.0;
        const float mu = (float)m, sg = (float)sqrt(var);
        // data = (data - mean) / std: finite iff every input is finite and std > 0
        const bool fin = isfinite(mu) && isfinite(sg) && sg > 0.0f;
        pa.mu[i] = mu; pa.sigma[i] = sg; pa.finite[i] = fin ? 1 : 0;
    }
}

// ------------------------------------------------------------------ first layer by linearity (FirstFuse, conv_gemm.cuh)
// Y[r][x][c] = sum_{kh,kw} w[kh][kw][c] * mspec[f0 + r + kh][x + kw] in float64, for the frames a batch of patches
// covers, stored as the two-float number Yh + Yl (FirstFuse, conv_gemm.cuh); one thread = one (row, column) position
// and 4 channels, filter in shared memory.
__global__ void __launch_bounds__(256)
first_linear_kernel(const float *__restrict__ mspec, int ld, int64_t f0, int64_t rows, int64_t n_frames, int OW, int KH, int KW, int C,
                    const float *__restrict__ w, float *__restrict__ Yh, float *__restrict__ Yl)
{
    extern __shared__ __align__(16) float wsm[];               // [KH * KW][C]  (float64 weights in shared memory measured slower: 61 vs 47 us)
    for (int i = threadIdx.x; i < KH * KW * C; i += 256) wsm[i] = w[i];
    __syncthreads();
    const int CQ = C >> 2;
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;  // over [row][x][c / 4]
    if (i >= rows * OW * CQ) return;
    const int c4 = (int)(i % CQ);
    const int64_t rx = i / CQ;
    const int x = (int)(rx % OW);
    const int64_t r = rx / OW;
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    for (int kh = 0; kh < KH; ++kh) {
        const int64_t f = f0 + r + kh;
        if (f >= n_frames) continue;                            // rows past the last frame are never read by a patch
        const float *src = mspec + f * ld + x;
        for (int kw = 0; kw < KW; ++kw) {
            const double xv = (double)__ldg(src + kw);
            const float4 w4 = *reinterpret_cast<const float4 *>(wsm + (kh * KW + kw) * C + c4 * 4);
            acc[0] = fma(xv, (double)w4.x, acc[0]); acc[1] = fma(xv, (double)w4.y, acc[1]);
            acc[2] = fma(xv, (double)w4.z, acc[2]); acc[3] = fma(xv, (double)w4.w, acc[3]);
        }
    }
    float h[4], l[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) { h[q] = (float)acc[q]; l[q] = (float)(acc[q] - (double)h[q]); }
    const int64_t o = (r * OW + x) * (int64_t)C + c4 * 4;
    *reinterpret_cast<float4 *>(Yh + o) = make_float4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<float4 *>(Yl + o) = make_float4(l[0], l[1], l[2], l[3]);
}

// Per (patch, channel) coefficients of the fused first layer (FirstFuse): alpha = s_c / sigma_j rounded to float32,
// beta = (b_c s_c + t_c) - mu_j S_c alpha in float64 (from the ROUNDED alpha), stored as two floats.  coef[j][3][C].
__global__ void __launch_bounds__(256)
first_coef_kernel(const float *__restrict__ mu, const float *__restrict__ sigma, const double *__restrict__ S,
                  const float *__restrict__ bias, const float *__restrict__ pre_scale, const float *__restrict__ pre_shift,
                  int64_t n, int C, float *__restrict__ coef)
{
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= n * C) return;
    const int c = (int)(i % C);
    const int64_t j = i / C;
    const double s1 = pre_scale ? (double)pre_scale[c] : 1.0, t1 = pre_shift ? (double)pre_shift[c] : 0.0;
    const double b = bias ? (double)bias[c] : 0.0;
    const float alpha = (float)(s1 / (double)sigma[j]);
    const double beta = (b * s1 + t1) - (double)mu[j] * S[c] * (double)alpha;
    const float bh = (float)beta;
    float *dst = coef + j * 3 * C + c;
    dst[0] = alpha; dst[C] = bh; dst[2 * C] = (float)(beta - (double)bh);
}

// ------------------------------------------------------------------ max pooling (NHWC)
// One thread per lane T of the output, over [img][oh][ow][C / lane width]: one fp32 value (float), four fp32 values with
// 16-byte loads and stores (float4, C % 4 == 0), or four split-half words (uint4, the tensor between two fp16-split
// convolutions).  Words are compared on their decoded values hi + lo (exact in fp32) and the winning WORD is stored, so the value itself is
// unchanged.  NaN propagates like TF's max; the first maximum wins.  The pooling layers are pure HBM traffic (218 KB in /
// 53 KB out per patch for the first one).
template <typename T>
__global__ void __launch_bounds__(256)
maxpool_nhwc_kernel(const T *__restrict__ in, T *__restrict__ out, int64_t total, int H, int W, int CL,
                    int OH, int OW, int KH, int KW, int SH, int SW, int PT, int PL)
{
    constexpr int Q = sizeof(T) / sizeof(uint32_t);
    constexpr bool WORDS = std::is_same<T, uint4>::value;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int c = (int)(i % CL);
    int64_t r = i / CL;
    const int ow = (int)(r % OW); r /= OW;
    const int oh = (int)(r % OH);
    const int64_t img = r / OH;
    float bv[Q];
    uint32_t bw[Q];
#pragma unroll
    for (int q = 0; q < Q; ++q) { bv[q] = -INFINITY; bw[q] = iss_pack_split(-INFINITY); }
    for (int y = 0; y < KH; ++y) {
        const int ih = oh * SH - PT + y;
        if (ih < 0 || ih >= H) continue;
        for (int x = 0; x < KW; ++x) {
            const int iw = ow * SW - PL + x;
            if (iw < 0 || iw >= W) continue;
            const T v = __ldg(in + ((img * H + ih) * W + iw) * CL + c);
            const uint32_t *w = reinterpret_cast<const uint32_t *>(&v);
#pragma unroll
            for (int q = 0; q < Q; ++q) {
                if constexpr (WORDS) {
                    const float f = iss_unpack_split(w[q]);
                    if (f > bv[q] || f != f) { bv[q] = f; bw[q] = w[q]; }
                } else {
                    const float f = __uint_as_float(w[q]);
                    bv[q] = (f > bv[q] || f != f) ? f : bv[q];
                }
            }
        }
    }
    T res;
    uint32_t *rw = reinterpret_cast<uint32_t *>(&res);
#pragma unroll
    for (int q = 0; q < Q; ++q) rw[q] = WORDS ? bw[q] : __float_as_uint(bv[q]);
    out[i] = res;
}

// ------------------------------------------------------------------ softmax head + non-finite override
__global__ void __launch_bounds__(256)
softmax_head_kernel(const float *__restrict__ logits, const uint8_t *__restrict__ finite, int64_t n, int K,
                    int do_softmax, float *__restrict__ probs)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float *l = logits + i * K;
    float *p = probs + i * K;
    if (!finite[i]) {                                   // r[finite == False, :] = 0.5 (segmenter.py:175)
        for (int k = 0; k < K; ++k) p[k] = 0.5f;
        return;
    }
    if (!do_softmax) { for (int k = 0; k < K; ++k) p[k] = l[k]; return; }
    float mx = l[0];
    for (int k = 1; k < K; ++k) mx = fmaxf(mx, l[k]);
    float s = 0.f;
    float e[8];
    for (int k = 0; k < K; ++k) { e[k] = expf(l[k] - mx); s += e[k]; }
    for (int k = 0; k < K; ++k) p[k] = e[k] / s;
}

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

}  // namespace

extern "C" int iss_cnn_destroy(iss_cnn *cnn);

extern "C" int iss_cnn_create(iss_ctx *ctx, const iss_layer_desc *layers, int n_layers,
                              const float *h_blob, int64_t blob_len, int in_h, int in_w, iss_cnn **out)
{
    ISS_REQUIRE(ctx && layers && h_blob && out && n_layers > 0, ISS_ERR_INVALID, "iss_cnn_create: bad argument");
    ISS_REQUIRE(in_h == PATCH_H, ISS_ERR_UNSUPPORTED, "iss_cnn_create: patch height must be %d (segmenter.py:149)", PATCH_H);
    ISS_REQUIRE(in_w >= 1 && in_w <= ISS_NMEL, ISS_ERR_INVALID, "iss_cnn_create: in_w=%d", in_w);
    ISS_CUDA_OK(cudaSetDevice(ctx->device));
    iss_cnn *m = new iss_cnn();
    m->ctx = ctx; m->d_blob = nullptr; m->blob_len = blob_len; m->in_h = in_h; m->in_w = in_w;
    int h = in_h, w = in_w, c = 1;
    int64_t max_act = 0;
    double flops = 0;
    auto off_ok = [&](int64_t off, int64_t len) { return off >= 0 && off + len <= blob_len; };
    for (int i = 0; i < n_layers; ++i) {
        Layer L; L.d = layers[i]; L.in_h = h; L.in_w = w; L.in_c = c;
        const iss_layer_desc &d = L.d;
        bool ok = true;
        if (d.kind == ISS_LAYER_CONV2D || d.kind == ISS_LAYER_MAXPOOL) {
            ok = d.kh >= 1 && d.kw >= 1 && d.sh >= 1 && d.sw >= 1 && d.pad_top >= 0 && d.pad_left >= 0 &&
                 d.pad_bottom >= 0 && d.pad_right >= 0;
            if (ok) {
                L.out_h = (h + d.pad_top + d.pad_bottom - d.kh) / d.sh + 1;
                L.out_w = (w + d.pad_left + d.pad_right - d.kw) / d.sw + 1;
                ok = L.out_h >= 1 && L.out_w >= 1;
            }
            if (d.kind == ISS_LAYER_CONV2D) {
                ok = ok && d.cin == c && d.cout >= 1 && off_ok(d.w_off, (int64_t)d.kh * d.kw * d.cin * d.cout);
                L.out_c = d.cout;
            } else {
                L.out_c = c;
            }
        } else if (d.kind == ISS_LAYER_DENSE) {
            ok = d.cin == h * w * c && d.cout >= 1 && off_ok(d.w_off, (int64_t)d.cin * d.cout);
            L.out_h = 1; L.out_w = 1; L.out_c = d.cout;
        } else {
            ok = false;
        }
        if (ok && d.kind != ISS_LAYER_MAXPOOL) {
            if (d.flags & ISS_F_BIAS) ok = ok && off_ok(d.bias_off, d.cout);
            if (d.flags & ISS_F_AFFINE_PRE) ok = ok && off_ok(d.pre_scale_off, d.cout) && off_ok(d.pre_shift_off, d.cout);
            if (d.flags & ISS_F_AFFINE_POST) ok = ok && off_ok(d.post_scale_off, d.cout) && off_ok(d.post_shift_off, d.cout);
            if (d.flags & ISS_F_SOFTMAX) ok = ok && (i == n_layers - 1) && d.cout <= 8;
        }
        if (!ok) {
            delete m;
            iss_set_error("iss_cnn_create: layer %d (kind %d) inconsistent with input %dx%dx%d or blob", i, d.kind, h, w, c);
            return ISS_ERR_UNSUPPORTED;
        }
        h = L.out_h; w = L.out_w; c = L.out_c;
        flops += layer_flops(L);
        max_act = std::max<int64_t>(max_act, (int64_t)h * w * c);
        m->layers.push_back(L);
    }
    if (!(h == 1 && w == 1 && c <= 8)) {
        delete m;
        iss_set_error("iss_cnn_create: network must end in a Dense head with <= 8 classes (got %dx%dx%d)", h, w, c);
        return ISS_ERR_UNSUPPORTED;
    }
    m->n_classes = c; m->max_act = max_act; m->flops = flops;
    cudaError_t e = cudaMalloc(&m->d_blob, (size_t)blob_len * sizeof(float));
    if (e != cudaSuccess) { delete m; iss_set_error("cudaMalloc blob: %s", cudaGetErrorString(e)); return ISS_ERR_NOMEM; }
    e = cudaMemcpy(m->d_blob, h_blob, (size_t)blob_len * sizeof(float), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) { cudaFree(m->d_blob); delete m; iss_set_error("cudaMemcpy blob: %s", cudaGetErrorString(e)); return ISS_ERR_CUDA; }
    for (size_t i = 1; i < m->layers.size(); ++i) {          // layer 0 gathers from the log-mel rows (fp32 kernel)
        Layer &L = m->layers[i];
        const iss_layer_desc &d = L.d;
        if (d.kind == ISS_LAYER_MAXPOOL) continue;
        const int K = (d.kind == ISS_LAYER_DENSE) ? d.cin : d.kh * d.kw * d.cin;
        const int rc = iss_prepare_weights(h_blob + d.w_off, d.cin, K, d.cout, true, &L.wt);
        if (rc != ISS_OK) { iss_cnn_destroy(m); return rc; }
    }
    {   // S_c = sum of the first layer's taps (float64), for the fused first layer
        const iss_layer_desc &d0 = m->layers[0].d;
        if (d0.kind == ISS_LAYER_CONV2D && d0.cin == 1) {
            std::vector<double> S(d0.cout, 0.0);
            for (int t = 0; t < d0.kh * d0.kw; ++t)
                for (int c = 0; c < d0.cout; ++c) S[c] += (double)h_blob[d0.w_off + (int64_t)t * d0.cout + c];
            e = cudaMalloc(&m->d_first_S, sizeof(double) * d0.cout);
            if (e == cudaSuccess) e = cudaMemcpy(m->d_first_S, S.data(), sizeof(double) * d0.cout, cudaMemcpyHostToDevice);
            if (e != cudaSuccess) { iss_cnn_destroy(m); iss_set_error("first-layer sums: %s", cudaGetErrorString(e)); return ISS_ERR_CUDA; }
        }
    }
    *out = m;
    return ISS_OK;
}

extern "C" int iss_cnn_destroy(iss_cnn *cnn)
{
    if (!cnn) return ISS_OK;
    cudaSetDevice(cnn->ctx->device);
    for (cudaEvent_t ev : cnn->prof_ev) cudaEventDestroy(ev);
    for (Layer &L : cnn->layers) iss_free_weights(&L.wt);
    if (cnn->d_blob) cudaFree(cnn->d_blob);
    if (cnn->d_first_S) cudaFree(cnn->d_first_S);
    delete cnn;
    return ISS_OK;
}

extern "C" int iss_cnn_num_classes(const iss_cnn *cnn) { return cnn ? cnn->n_classes : -1; }
extern "C" double iss_cnn_flops_per_patch(const iss_cnn *cnn) { return cnn ? cnn->flops : 0.0; }

namespace {
// rows of the two-float first-layer map a batch of B patches may need (3x the contiguous case; batches whose
// patches are spread wider fall back to the un-fused first layer) and its size in bytes (0: no fusion possible)
int64_t first_y_rows(int64_t B) { return 3 * (PATCH_HOP * B + PATCH_H); }
size_t first_y_bytes(const iss_cnn *cnn, int64_t B)
{
    if (!cnn->d_first_S || cnn->layers.size() < 2) return 0;
    const Layer &L0 = cnn->layers[0];
    return 2 * align_up((size_t)first_y_rows(B) * L0.out_w * L0.out_c * sizeof(float), 256) +        // Yh, Yl
           align_up((size_t)B * 3 * L0.out_c * sizeof(float), 256);                                   // per-patch coefficients
}
}  // namespace

extern "C" int64_t iss_cnn_workspace_bytes(const iss_cnn *cnn, int64_t n, int n_seg)
{
    if (!cnn || n < 0 || n_seg < 0) return -1;
    const int64_t B = std::min<int64_t>(std::max<int64_t>(n, 1), CNN_BATCH);
    int64_t bytes = 0;
    bytes += align_up((size_t)n * 4, 256) * 3;            // row0, mu, sigma
    bytes += align_up((size_t)n, 256);                     // finite
    bytes += align_up((size_t)n * 8 * 4, 256);             // logits [n][<=8]
    bytes += 2 * align_up((size_t)B * cnn->max_act * 4, 256);
    bytes += align_up((size_t)(n_seg + 1) * sizeof(PatchRange), 256) + align_up((size_t)(n_seg + 1) * 8, 256);   // range tables
    bytes += first_y_bytes(cnn, B);                                                               // float64 map of the fused first layer
    return bytes;
}

namespace {

template <typename T>
void launch_pool(const Layer &L, const float *in, float *out, int64_t nb, cudaStream_t st)
{
    constexpr int Q = sizeof(T) / sizeof(uint32_t);
    const iss_layer_desc &d = L.d;
    const int64_t total = nb * L.out_h * L.out_w * L.out_c / Q;
    maxpool_nhwc_kernel<T><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(
        reinterpret_cast<const T *>(in), reinterpret_cast<T *>(out), total, L.in_h, L.in_w, L.in_c / Q,
        L.out_h, L.out_w, d.kh, d.kw, d.sh, d.sw, d.pad_top, d.pad_left);
}

// How iss_cnn_forward runs a layer
enum class Step {
    FOLDED_POOL,        // 2x2 / stride-2 pooling taken in the next convolution's operand fill: nothing runs
    POOL,               // maxpool_nhwc_kernel
    CONV,               // iss_launch_conv, unless the batch folds layer 0 into layer 1
};

struct LayerPlan {
    Step step;
    void (*pool)(const Layer &, const float *, float *, int64_t, cudaStream_t);     // POOL: launch_pool of the lane type
    // CONV: all but in, out, M and `first` of the batch; layer 0 holds the log-mel source of the whole call.  in_packed /
    // out_packed are the activation formats, pool_h / pool_w the dims of a pooling folded into this layer.
    ConvArgs a;
};

// The kernel and activation formats of every layer for one call of iss_cnn_forward, from the GEMM mode, the switches
// ISS_B200_FUSE_POOL / ISS_B200_FUSE_FIRST ("0": pooling / first layer as their own kernels) and the profiled layer,
// all of which may change between calls.  *fuse_first: layer 0 may be folded into layer 1 (first_map: the workspace
// holds the fused first layer's map and the ranges ascend), decided per batch by the frames its patches span.
int plan_forward(const iss_cnn *cnn, int mode, const float *mspec, int ld, const PatchArrays &pa, bool first_map,
                 std::vector<LayerPlan> &plan, bool *fuse_first)
{
    const char *e = getenv("ISS_B200_FUSE_POOL");
    const bool fuse_pool = !(e && e[0] == '0');
    e = getenv("ISS_B200_FUSE_FIRST");
    const bool fuse_first_on = !(e && e[0] == '0');
    const size_t n = cnn->layers.size();
    plan.assign(n, LayerPlan{});
    for (size_t li = 0; li < n; ++li) {
        const Layer &Lr = cnn->layers[li];
        const iss_layer_desc &d = Lr.d;
        if (d.kind == ISS_LAYER_MAXPOOL) continue;
        const float *blob = cnn->d_blob;
        ConvArgs &a = plan[li].a;
        a.w = blob + d.w_off;
        a.bias = (d.flags & ISS_F_BIAS) ? blob + d.bias_off : nullptr;
        a.pre_scale = (d.flags & ISS_F_AFFINE_PRE) ? blob + d.pre_scale_off : nullptr;
        a.pre_shift = (d.flags & ISS_F_AFFINE_PRE) ? blob + d.pre_shift_off : nullptr;
        a.post_scale = (d.flags & ISS_F_AFFINE_POST) ? blob + d.post_scale_off : nullptr;
        a.post_shift = (d.flags & ISS_F_AFFINE_POST) ? blob + d.post_shift_off : nullptr;
        a.flags = d.flags & ~ISS_F_SOFTMAX;
        a.wt = Lr.wt;
        a.N = d.cout;
        if (d.kind == ISS_LAYER_DENSE) {
            a.K = d.cin; a.H = 1; a.W = 1; a.C = d.cin; a.OH = 1; a.OW = 1;
            a.KH = 1; a.KW = 1; a.SH = 1; a.SW = 1; a.PT = 0; a.PL = 0;
        } else {
            a.K = d.kh * d.kw * d.cin;
            a.H = Lr.in_h; a.W = Lr.in_w; a.C = Lr.in_c; a.OH = Lr.out_h; a.OW = Lr.out_w;
            a.KH = d.kh; a.KW = d.kw; a.SH = d.sh; a.SW = d.sw; a.PT = d.pad_top; a.PL = d.pad_left;
        }
        if (li == 0) { a.in = mspec; a.ld = ld; a.row0 = pa.row0; a.mu = pa.mu; a.sigma = pa.sigma; }
    }
    auto f16 = [&](const ConvArgs &a) { return iss_conv_is_f16(iss_conv_kernel(a, mode)); };
    // does compute layer j run on engine 3 when handed split-half words?
    auto reads_packed = [&](size_t j) { ConvArgs a = plan[j].a; a.in_packed = 1; return f16(a); };

    bool packed = false;                                     // format of the activation the next layer reads
    int pool_h = 0, pool_w = 0;                              // un-pooled dims of a pooling folded into the next layer
    for (size_t li = 0; li < n; ++li) {
        const Layer &Lr = cnn->layers[li];
        const iss_layer_desc &d = Lr.d;
        LayerPlan &P = plan[li];
        if (d.kind == ISS_LAYER_MAXPOOL) {
            ISS_REQUIRE(li > 0, ISS_ERR_UNSUPPORTED, "iss_cnn_forward: pooling as first layer is not supported");
            // 2x2 / stride-2 'valid' pooling over split-half words in front of a convolution engine 3 takes with the
            // pooling folded in: the maximum is taken in its operand fill (conv_gemm_tc.cu, LD_POOL)
            const Layer *Nx = li + 1 < n ? &cnn->layers[li + 1] : nullptr;
            if (packed && fuse_pool && (int)li != cnn->prof_layer && Nx && d.kh == 2 && d.kw == 2 && d.sh == 2 && d.sw == 2 &&
                d.pad_top == 0 && d.pad_left == 0 && d.pad_bottom == 0 && d.pad_right == 0 &&
                Nx->d.kind == ISS_LAYER_CONV2D && Nx->d.pad_bottom == 0 && Nx->d.pad_right == 0) {
                ConvArgs a = plan[li + 1].a;
                a.in_packed = 1; a.pool_h = Lr.in_h; a.pool_w = Lr.in_w;
                if (f16(a)) { P.step = Step::FOLDED_POOL; pool_h = Lr.in_h; pool_w = Lr.in_w; continue; }
            }
            P.step = Step::POOL;
            P.pool = packed ? launch_pool<uint4> : Lr.in_c % 4 == 0 ? launch_pool<float4> : launch_pool<float>;
            continue;
        }
        ConvArgs &a = P.a;
        a.in_packed = packed;
        a.pool_h = pool_h; a.pool_w = pool_w;
        pool_h = pool_w = 0;
        // split-half output iff the next compute layer reads it on engine 3; pooling layers in between keep the
        // format (the word lane of the pooling kernel moves 4 channels per thread)
        size_t j = li + 1;
        bool pools_vec4 = true;
        for (; j < n && cnn->layers[j].d.kind == ISS_LAYER_MAXPOOL; ++j) pools_vec4 = pools_vec4 && cnn->layers[j].in_c % 4 == 0;
        const bool next_packed = j < n && pools_vec4 && reads_packed(j);
        ISS_REQUIRE(li > 0 || d.kind == ISS_LAYER_CONV2D, ISS_ERR_UNSUPPORTED, "iss_cnn_forward: first layer must be Conv2D");
        P.step = Step::CONV;
        a.out_packed = next_packed && iss_conv_writes_words(iss_conv_kernel(a, mode));
        if (li == 0) {
            // the fused first layer (FirstFuse, conv_gemm.cuh): the direct kernel's shape without padding / stride, in
            // layer 1's slab-kernel operand fill
            *fuse_first = false;
            if (a.out_packed && fuse_first_on && first_map && d.sh == 1 && d.sw == 1 && d.pad_top == 0 && d.pad_left == 0 &&
                d.pad_bottom == 0 && d.pad_right == 0 && !(d.flags & ISS_F_SIGMOID) && cnn->layers[1].d.kind == ISS_LAYER_CONV2D &&
                cnn->layers[1].d.pad_bottom == 0 && cnn->layers[1].d.pad_right == 0) {
                const FirstFuse probe = {};
                ConvArgs a1 = plan[1].a;
                a1.in_packed = 1; a1.first = &probe;
                *fuse_first = f16(a1);
            }
        }
        packed = a.out_packed;
    }
    return ISS_OK;
}

}  // namespace

// The forward pass over n_rec recordings packed in one log-mel buffer of `rows` rows: recording r is rows
// [h_row_off[r], h_row_off[r] + h_len[r]), and range s covers padded patches [h_seg_start[s], h_seg_stop[s]) of recording
// h_seg_rec[s] (h_seg_rec == nullptr: all ranges are of recording 0).  The edge flags apply to every recording.
static int cnn_forward(iss_ctx *ctx, iss_cnn *cnn, const float *d_mspec, int64_t rows, int ld, int edge_left, int edge_right,
                       const int64_t *h_row_off, const int64_t *h_len, int n_rec, const int32_t *h_seg_rec,
                       const int32_t *h_seg_start, const int32_t *h_seg_stop, int n_seg,
                       float *d_probs, void *d_work, int64_t work_bytes, void *stream)
{
    ISS_REQUIRE(ctx && cnn, ISS_ERR_INVALID, "iss_cnn_forward: NULL handle");
    ISS_REQUIRE(ld >= cnn->in_w, ISS_ERR_INVALID, "iss_cnn_forward: ld=%d < nmel=%d", ld, cnn->in_w);
    if (n_seg <= 0) return ISS_OK;
    ISS_REQUIRE(h_seg_start && h_seg_stop, ISS_ERR_INVALID, "iss_cnn_forward: NULL segment arrays");
    ISS_REQUIRE(rows < (1ll << 31), ISS_ERR_INVALID, "iss_cnn_forward: %lld log-mel rows do not fit 32-bit row indices", (long long)rows);
    for (int r = 0; r < n_rec; ++r) {
        const int64_t L = h_len[r];
        ISS_REQUIRE(L >= PATCH_H, ISS_ERR_INVALID, "iss_cnn_forward: L=%lld < %d frames (pad short inputs first, segmenter.py:60-65)", (long long)L, PATCH_H);
        ISS_REQUIRE(h_row_off[r] >= 0 && h_row_off[r] + L <= rows, ISS_ERR_INVALID,
                    "iss_cnn_forward: recording %d = rows [%lld,%lld) outside [0,%lld)", r, (long long)h_row_off[r],
                    (long long)(h_row_off[r] + L), (long long)rows);
    }
    ISS_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = iss_stream(stream);
    std::vector<int64_t> off(n_seg + 1);
    std::vector<PatchRange> rng(n_seg + 1);
    int64_t n = 0;
    for (int s = 0; s < n_seg; ++s) {
        const int rec = h_seg_rec ? h_seg_rec[s] : 0;
        ISS_REQUIRE(rec >= 0 && rec < n_rec, ISS_ERR_INVALID, "iss_cnn_forward: range %d names recording %d of %d", s, rec, n_rec);
        const int64_t L = h_len[rec];
        const int64_t U = (L - PATCH_H) / PATCH_HOP + 1;                      // un-replicated windows
        const int64_t P = (edge_left ? PATCH_LFILL : 0) + U + (edge_right ? (PATCH_LFILL - 1 + (L % 2)) : 0);
        ISS_REQUIRE(h_seg_start[s] >= 0 && h_seg_stop[s] >= h_seg_start[s] && h_seg_stop[s] <= P, ISS_ERR_INVALID,
                    "iss_cnn_forward: range %d = [%d,%d) outside [0,%lld)", s, h_seg_start[s], h_seg_stop[s], (long long)P);
        rng[s] = PatchRange{h_row_off[rec], U, h_seg_start[s]};
        off[s] = n; n += h_seg_stop[s] - h_seg_start[s];
    }
    off[n_seg] = n;
    rng[n_seg] = PatchRange{0, 0, 0};
    if (n == 0) return ISS_OK;
    ISS_REQUIRE(d_mspec && d_probs && d_work, ISS_ERR_INVALID, "iss_cnn_forward: NULL buffer");
    ISS_REQUIRE(work_bytes >= iss_cnn_workspace_bytes(cnn, n, n_seg), ISS_ERR_INVALID,
                "iss_cnn_forward: workspace %lld < required %lld", (long long)work_bytes, (long long)iss_cnn_workspace_bytes(cnn, n, n_seg));

    // ---- carve the workspace ----
    const int64_t B = std::min<int64_t>(n, CNN_BATCH);
    uint8_t *p = reinterpret_cast<uint8_t *>(d_work);
    size_t o = 0;
    PatchArrays pa;
    pa.row0 = reinterpret_cast<int32_t *>(p + o); o += align_up((size_t)n * 4, 256);
    pa.mu = reinterpret_cast<float *>(p + o);     o += align_up((size_t)n * 4, 256);
    pa.sigma = reinterpret_cast<float *>(p + o);  o += align_up((size_t)n * 4, 256);
    pa.finite = p + o;                            o += align_up((size_t)n, 256);
    float *logits = reinterpret_cast<float *>(p + o); o += align_up((size_t)n * 8 * 4, 256);
    float *act[2];
    act[0] = reinterpret_cast<float *>(p + o);    o += align_up((size_t)B * cnn->max_act * 4, 256);
    act[1] = reinterpret_cast<float *>(p + o);    o += align_up((size_t)B * cnn->max_act * 4, 256);
    PatchRange *d_ranges = reinterpret_cast<PatchRange *>(p + o); o += align_up((size_t)(n_seg + 1) * sizeof(PatchRange), 256);
    int64_t *d_seg_off = reinterpret_cast<int64_t *>(p + o);   o += align_up((size_t)(n_seg + 1) * 8, 256);
    float *d_first_yh = nullptr, *d_first_yl = nullptr, *d_first_coef = nullptr;                // fused first layer (FirstFuse)
    if (first_y_bytes(cnn, B)) {
        const Layer &L0 = cnn->layers[0];
        const size_t plane = align_up((size_t)first_y_rows(B) * L0.out_w * L0.out_c * sizeof(float), 256);
        d_first_yh = reinterpret_cast<float *>(p + o); d_first_yl = reinterpret_cast<float *>(p + o + plane);
        d_first_coef = reinterpret_cast<float *>(p + o + 2 * plane);
        o += first_y_bytes(cnn, B);
    }
    // host copy of patch_index_kernel's arithmetic: first log-mel frame of patch i (for the span of a batch)
    auto host_row0 = [&](int64_t i) -> int64_t {
        int lo = 0, hi = n_seg;
        while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (off[mid] <= i) lo = mid; else hi = mid; }
        return patch_row0(rng[lo], h_seg_start[lo] + (i - off[lo]), edge_left, edge_right);
    };
    // the fused first layer needs patch rows that never decrease: ranges of one recording ascend, and a range of another
    // recording starts at or after the last row of the range before it
    bool ranges_ascending = true;
    for (int s = 1; s < n_seg; ++s) {
        const bool same = !h_seg_rec || h_seg_rec[s] == h_seg_rec[s - 1];
        ranges_ascending = ranges_ascending && (same ? h_seg_start[s] >= h_seg_stop[s - 1]
                                                     : (off[s] == 0 || off[s] == n || host_row0(off[s]) >= host_row0(off[s] - 1)));
    }
    const int mode = iss_get_gemm_mode();
    std::vector<LayerPlan> plan;
    bool fuse_first = false;
    const int prc = plan_forward(cnn, mode, d_mspec, ld, pa, d_first_yh && ranges_ascending, plan, &fuse_first);
    if (prc != ISS_OK) return prc;
    ISS_CUDA_OK(cudaMemcpyAsync(d_ranges, rng.data(), sizeof(PatchRange) * n_seg, cudaMemcpyHostToDevice, st));
    ISS_CUDA_OK(cudaMemcpyAsync(d_seg_off, off.data(), sizeof(int64_t) * (n_seg + 1), cudaMemcpyHostToDevice, st));

    patch_index_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_ranges, d_seg_off, n_seg, n, edge_left, edge_right, pa.row0);
    patch_stats_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, st>>>(d_mspec, ld, cnn->in_w, n, pa);
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch(2);

    const int K = cnn->n_classes;
    for (int64_t b0 = 0; b0 < n; b0 += B) {
        const int64_t nb = std::min<int64_t>(B, n - b0);
        const float *cur = nullptr;
        int which = 0;
        FirstFuse ffuse = {};                                    // set by layer 0 when this batch folds it into layer 1
        bool first_fused = false;
        for (size_t li = 0; li < cnn->layers.size(); ++li) {
            const Layer &Lr = cnn->layers[li];
            const iss_layer_desc &d = Lr.d;
            const LayerPlan &P = plan[li];
            if (P.step == Step::FOLDED_POOL) continue;
            const bool last = (li + 1 == cnn->layers.size());
            float *dst = last ? (logits + b0 * K) : act[which];
            const bool prof = ((int)li == cnn->prof_layer);
            if (prof) {
                if (cnn->prof_used + 2 > cnn->prof_ev.size()) {
                    for (int q = 0; q < 2; ++q) {
                        cudaEvent_t ev;
                        ISS_CUDA_OK(cudaEventCreate(&ev));
                        cnn->prof_ev.push_back(ev);
                    }
                }
                ISS_CUDA_OK(cudaEventRecord(cnn->prof_ev[cnn->prof_used], st));
            }
            if (P.step == Step::POOL) {
                P.pool(Lr, cur, dst, nb, st);
                ISS_CUDA_OK(cudaGetLastError());
                iss_count_launch();
            } else {
                ConvArgs a = P.a;
                a.out = dst;
                a.M = nb * a.OH * a.OW;
                if (a.row0) { a.row0 += b0; a.mu += b0; a.sigma += b0; }
                else a.in = cur;
                if (li == 0 && fuse_first) {
                    // the float64 map of the first layer covers the frames this batch's patches span, if few enough
                    const int64_t f_first = host_row0(b0), f_last = host_row0(b0 + nb - 1);
                    const int64_t map_rows = f_last - f_first + Lr.out_h;
                    if (map_rows <= first_y_rows(B)) {
                        const int64_t work = map_rows * Lr.out_w * (d.cout >> 2);
                        first_linear_kernel<<<(unsigned)((work + 255) / 256), 256, (size_t)d.kh * d.kw * d.cout * sizeof(float), st>>>(
                            d_mspec, ld, f_first, map_rows, rows, Lr.out_w, d.kh, d.kw, d.cout, a.w, d_first_yh, d_first_yl);
                        first_coef_kernel<<<(unsigned)((nb * d.cout + 255) / 256), 256, 0, st>>>(
                            a.mu, a.sigma, cnn->d_first_S, a.bias, a.pre_scale, a.pre_shift, nb, d.cout, d_first_coef);
                        ISS_CUDA_OK(cudaGetLastError());
                        iss_count_launch(2);
                        ffuse.Yh = d_first_yh; ffuse.Yl = d_first_yl; ffuse.y_f0 = f_first; ffuse.y_rows = map_rows;
                        ffuse.row0 = a.row0; ffuse.coef = d_first_coef;
                        ffuse.post_scale = a.post_scale; ffuse.post_shift = a.post_shift; ffuse.flags = a.flags; ffuse.n_img = nb;
                        first_fused = true;                      // nothing stored: layer 1 reads the map
                    }
                }
                if (li == 1 && first_fused) { a.first = &ffuse; a.in = nullptr; }
                if (!(li == 0 && first_fused)) {
                    const int rc = iss_launch_conv(a, mode, st);
                    if (rc != ISS_OK) return rc;
                }
            }
            if (prof) {
                ISS_CUDA_OK(cudaEventRecord(cnn->prof_ev[cnn->prof_used + 1], st));
                cnn->prof_used += 2;
                cnn->prof_flops += nb * layer_flops(Lr);
            }
            cur = dst;
            which ^= 1;
        }
    }
    const Layer &head = cnn->layers.back();
    softmax_head_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(logits, pa.finite, n, K,
        (head.d.flags & ISS_F_SOFTMAX) ? 1 : 0, d_probs);
    ISS_CUDA_OK(cudaGetLastError());
    iss_count_launch();
    return ISS_OK;
}

extern "C" int iss_cnn_forward(iss_ctx *ctx, iss_cnn *cnn, const float *d_mspec, int64_t L, int ld,
                               int edge_left, int edge_right,
                               const int32_t *h_seg_start, const int32_t *h_seg_stop, int n_seg,
                               float *d_probs, void *d_work, int64_t work_bytes, void *stream)
{
    const int64_t zero = 0;
    return cnn_forward(ctx, cnn, d_mspec, L, ld, edge_left, edge_right, &zero, &L, 1, nullptr, h_seg_start, h_seg_stop, n_seg,
                       d_probs, d_work, work_bytes, stream);
}

extern "C" int iss_cnn_forward_multi(iss_ctx *ctx, iss_cnn *cnn, const float *d_mspec, int64_t rows, int ld,
                                     const int64_t *h_row_off, const int64_t *h_len, int n_rec,
                                     const int32_t *h_seg_rec, const int32_t *h_seg_start, const int32_t *h_seg_stop, int n_seg,
                                     float *d_probs, void *d_work, int64_t work_bytes, void *stream)
{
    ISS_REQUIRE(n_rec >= 1 && h_row_off && h_len && h_seg_rec, ISS_ERR_INVALID, "iss_cnn_forward_multi: bad recording arguments");
    return cnn_forward(ctx, cnn, d_mspec, rows, ld, 1, 1, h_row_off, h_len, n_rec, h_seg_rec, h_seg_start, h_seg_stop, n_seg,
                       d_probs, d_work, work_bytes, stream);
}

extern "C" int iss_cnn_profile(iss_cnn *cnn, int layer)
{
    ISS_REQUIRE(cnn, ISS_ERR_INVALID, "iss_cnn_profile: NULL");
    ISS_REQUIRE(layer >= -1 && layer < (int)cnn->layers.size(), ISS_ERR_INVALID, "iss_cnn_profile: layer %d", layer);
    cnn->prof_layer = layer;
    cnn->prof_used = 0;
    cnn->prof_flops = 0;
    return ISS_OK;
}

extern "C" int iss_cnn_profile_read(iss_cnn *cnn, double *total_ms, int64_t *launches, double *flops)
{
    ISS_REQUIRE(cnn && total_ms && launches && flops, ISS_ERR_INVALID, "iss_cnn_profile_read: NULL");
    ISS_CUDA_OK(cudaSetDevice(cnn->ctx->device));
    double t = 0;
    for (size_t i = 0; i + 1 < cnn->prof_used; i += 2) {
        ISS_CUDA_OK(cudaEventSynchronize(cnn->prof_ev[i + 1]));
        float ms = 0;
        ISS_CUDA_OK(cudaEventElapsedTime(&ms, cnn->prof_ev[i], cnn->prof_ev[i + 1]));
        t += ms;
    }
    *total_ms = t; *launches = (int64_t)(cnn->prof_used / 2); *flops = cnn->prof_flops;
    cnn->prof_used = 0; cnn->prof_flops = 0;
    return ISS_OK;
}

extern "C" int iss_cnn_num_layers(const iss_cnn *cnn) { return cnn ? (int)cnn->layers.size() : -1; }

extern "C" double iss_cnn_layer_flops(const iss_cnn *cnn, int layer)
{
    if (!cnn || layer < 0 || layer >= (int)cnn->layers.size()) return 0.0;
    return layer_flops(cnn->layers[layer]);
}
