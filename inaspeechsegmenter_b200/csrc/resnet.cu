// resnet.cu -- K5: VBx ResNet101 x-vector extractor forward (eval mode).
//
// Reference semantics: ResNet.forward (inaSpeechSegmenter/resnet.py:115-130) for
// ResNet101 = Bottleneck x [3,4,23,3], planes 32/64/128/256 (x4 expansion), strides
// 1/2/2/2 (:99-102,:133-135); Bottleneck (:48-75): 1x1 -> 3x3(stride) -> 1x1, BatchNorm
// after each, ReLU after the first two, shortcut 1x1(stride)+BN when the shape
// changes, add, ReLU; statistics pooling mean / sqrt(E[x^2]-E[x]^2+1e-10) over time
// (:123-125), flatten, Linear (:126-129).  Called once per 144-frame window by
// VBxExtractor (vbx_segmenter.py:222-243, batch 1 in the reference); here windows are
// batched, each keeping its own zero padding (a fully-convolutional pass over the
// recording would NOT be equivalent).
//
// Layout: activations NHWC float32 with H = mel band (64), W = time (T), so every
// convolution is the implicit GEMM of conv_gemm.cu; BatchNorm is folded into the
// epilogue's per-channel affine, the residual add + ReLU are fused into the last 1x1
// convolution of each block.
#include <math.h>
#include <stdlib.h>
#include <vector>

#include "conv_gemm.cuh"

namespace {

struct RConv {
    int kh, kw, stride, pad, cin, cout;
    int64_t w_off, scale_off, shift_off;
    TcWeights wt;
};

struct RBlock {
    RConv c1, c2, c3, sc;
    bool has_sc;
};

__global__ void __launch_bounds__(256)
window_gather_kernel(const float *__restrict__ fea, const int32_t *__restrict__ win_start, int n_win, int T, int F,
                     float *__restrict__ out)
{
    // out[w][f][t] = fea[(start_w + t) * F + f]   (fea.transpose(), vbx_segmenter.py:265)
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t total = (int64_t)n_win * F * T;
    if (i >= total) return;
    const int t = (int)(i % T);
    const int f = (int)((i / T) % F);
    const int w = (int)(i / ((int64_t)T * F));
    out[i] = fea[((int64_t)win_start[w] + t) * F + f];
}

__global__ void __launch_bounds__(256)
stat_pool_kernel(const float *__restrict__ in, int n_win, int H, int W, int C, float *__restrict__ pooled)
{
    // in: [w][h][t][c];  pooled[w][c*H + h] = mean_t, pooled[w][C*H + c*H + h] = std_t
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;       // over (w, h, c), c fastest
    if (i >= (int64_t)n_win * H * C) return;
    const int c = (int)(i % C);
    const int h = (int)((i / C) % H);
    const int w = (int)(i / ((int64_t)C * H));
    const float *p = in + (((int64_t)w * H + h) * W) * C + c;
    float s1 = 0.f, s2 = 0.f;
    for (int t = 0; t < W; ++t) { const float v = p[(int64_t)t * C]; s1 += v; s2 += v * v; }
    const float mean = s1 / (float)W, msq = s2 / (float)W;
    float *o = pooled + (int64_t)w * 2 * C * H;
    o[c * H + h] = mean;
    // msq - mean^2 of a (near-)constant channel rounds to either side of 0: clamped, so that the std is sqrt(1e-10) and not
    // NaN; the NaN-propagating max (iss_relu) keeps a non-finite activation non-finite
    o[C * H + c * H + h] = sqrtf(iss_relu(msq - mean * mean) + 1e-10f);
}

}  // namespace

struct iss_resnet {
    iss_ctx *ctx;
    float *d_blob;
    int64_t blob_len;
    int m, feat_dim, embed_dim;
    RConv stem;
    std::vector<RBlock> blocks;
    int64_t emb_w_off, emb_b_off;
    int c_final, h_final;
    TcWeights emb_wt;
};

namespace {

int out_dim(int x, int k, int s, int p) { return (x + 2 * p - k) / s + 1; }

// walks the architecture; returns blob length; fills net if non-null
int64_t build_plan(int m, int feat_dim, int embed_dim, const int *nb, iss_resnet *net)
{
    int64_t off = 0;
    auto mk = [&](int k, int stride, int pad, int cin, int cout) {
        RConv c;
        c.kh = k; c.kw = k; c.stride = stride; c.pad = pad; c.cin = cin; c.cout = cout;
        c.w_off = off; off += (int64_t)k * k * cin * cout;
        c.scale_off = off; off += cout;
        c.shift_off = off; off += cout;
        return c;
    };
    RConv stem = mk(3, 1, 1, 1, m);
    if (net) { net->stem = stem; net->blocks.clear(); }
    int inp = m, h = feat_dim;
    const int strides[4] = {1, 2, 2, 2};
    for (int li = 0; li < 4; ++li) {
        const int planes = m << li;
        for (int b = 0; b < nb[li]; ++b) {
            const int s = (b == 0) ? strides[li] : 1;
            RBlock blk;
            blk.c1 = mk(1, 1, 0, inp, planes);
            blk.c2 = mk(3, s, 1, planes, planes);
            blk.c3 = mk(1, 1, 0, planes, 4 * planes);
            blk.has_sc = (s != 1 || inp != 4 * planes);
            if (blk.has_sc) blk.sc = mk(1, s, 0, inp, 4 * planes);
            if (net) net->blocks.push_back(blk);
            inp = 4 * planes;
            h = out_dim(h, 3, s, 1);
        }
    }
    if (net) { net->emb_w_off = off; net->c_final = inp; net->h_final = h; }
    off += (int64_t)2 * inp * h * embed_dim;
    if (net) net->emb_b_off = off;
    off += embed_dim;
    return off;
}

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

int64_t max_act_per_window(const iss_resnet *net, int T, double *flops)
{
    // largest activation (floats) any buffer must hold for one window; also counts FLOPs
    int h = net->feat_dim, w = T;
    int64_t mx = (int64_t)h * w * net->m;
    double fl = 2.0 * h * w * 9.0 * net->m;
    for (const RBlock &b : net->blocks) {
        const int s = b.c2.stride;
        const int h2 = out_dim(h, 3, s, 1), w2 = out_dim(w, 3, s, 1);
        mx = std::max<int64_t>(mx, (int64_t)h * w * b.c1.cout);
        mx = std::max<int64_t>(mx, (int64_t)h2 * w2 * b.c3.cout);
        fl += 2.0 * h * w * (double)b.c1.cin * b.c1.cout;
        fl += 2.0 * h2 * w2 * 9.0 * b.c2.cin * b.c2.cout;
        fl += 2.0 * h2 * w2 * (double)b.c3.cin * b.c3.cout;
        if (b.has_sc) fl += 2.0 * h2 * w2 * (double)b.sc.cin * b.sc.cout;
        h = h2; w = w2;
    }
    fl += 2.0 * 2.0 * net->c_final * net->h_final * net->embed_dim;
    if (flops) *flops = fl;
    return mx;
}

// windows per sweep: 256 (layer4 then has 256*8*18/128 = 288 M-tiles; measured 101 TFLOP/s against 97 at 128 and 92 at
// 64 windows, gpurun_out r02j); ISS_B200_RES_BATCH: experiments, read once
static int res_batch()
{
    static const int b = [] { const char *e = getenv("ISS_B200_RES_BATCH"); const int v = e ? atoi(e) : 0; return v >= 8 && v <= 1024 ? v : 256; }();
    return b;
}
#define RES_BATCH res_batch()

}  // namespace

extern "C" int64_t iss_resnet_blob_len(int m_channels, int feat_dim, int embed_dim, const int *num_blocks)
{
    if (!num_blocks || m_channels < 1 || feat_dim < 8 || embed_dim < 1) return -1;
    return build_plan(m_channels, feat_dim, embed_dim, num_blocks, nullptr);
}

extern "C" int iss_resnet_destroy(iss_resnet *net);

extern "C" int iss_resnet_create(iss_ctx *ctx, const float *h_blob, int64_t blob_len, int m_channels, int feat_dim,
                                 int embed_dim, const int *num_blocks, iss_resnet **out)
{
    ISS_REQUIRE(ctx && h_blob && num_blocks && out, ISS_ERR_INVALID, "iss_resnet_create: NULL argument");
    ISS_REQUIRE(m_channels % 8 == 0 && feat_dim % 8 == 0, ISS_ERR_UNSUPPORTED, "iss_resnet_create: m_channels and feat_dim must be multiples of 8");
    ISS_CUDA_OK(cudaSetDevice(ctx->device));
    iss_resnet *net = new iss_resnet();
    net->ctx = ctx; net->d_blob = nullptr; net->m = m_channels; net->feat_dim = feat_dim; net->embed_dim = embed_dim;
    const int64_t need = build_plan(m_channels, feat_dim, embed_dim, num_blocks, net);
    if (need != blob_len) {
        delete net;
        iss_set_error("iss_resnet_create: blob has %lld floats, architecture needs %lld", (long long)blob_len, (long long)need);
        return ISS_ERR_INVALID;
    }
    net->blob_len = blob_len;
    cudaError_t e = cudaMalloc(&net->d_blob, (size_t)blob_len * sizeof(float));
    if (e != cudaSuccess) { delete net; iss_set_error("cudaMalloc resnet blob: %s", cudaGetErrorString(e)); return ISS_ERR_NOMEM; }
    e = cudaMemcpy(net->d_blob, h_blob, (size_t)blob_len * sizeof(float), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) { cudaFree(net->d_blob); delete net; iss_set_error("cudaMemcpy resnet blob: %s", cudaGetErrorString(e)); return ISS_ERR_CUDA; }
    auto prep = [&](RConv &c) { return iss_prepare_weights(h_blob + c.w_off, c.cin, c.kh * c.kw * c.cin, c.cout, true, &c.wt); };
    int prc = ISS_OK;
    for (RBlock &b : net->blocks) {
        if (prc == ISS_OK) prc = prep(b.c1);
        if (prc == ISS_OK) prc = prep(b.c2);
        if (prc == ISS_OK) prc = prep(b.c3);
        if (prc == ISS_OK && b.has_sc) prc = prep(b.sc);
    }
    if (prc == ISS_OK) {
        // the embedding stays on engine 2 in every mode: no engine-3 image
        const int K = 2 * net->c_final * net->h_final;
        prc = iss_prepare_weights(h_blob + net->emb_w_off, K, K, net->embed_dim, false, &net->emb_wt);
    }
    if (prc != ISS_OK) { iss_resnet_destroy(net); return prc; }
    *out = net;
    return ISS_OK;
}

extern "C" int iss_resnet_destroy(iss_resnet *net)
{
    if (!net) return ISS_OK;
    cudaSetDevice(net->ctx->device);
    if (net->d_blob) cudaFree(net->d_blob);
    iss_free_weights(&net->emb_wt);
    for (RBlock &b : net->blocks)
        for (RConv *c : {&b.c1, &b.c2, &b.c3, &b.sc}) iss_free_weights(&c->wt);
    delete net;
    return ISS_OK;
}

extern "C" double iss_resnet_flops_per_window(const iss_resnet *net, int win_len)
{
    if (!net || win_len < 1) return 0.0;
    double fl = 0;
    max_act_per_window(net, win_len, &fl);
    return fl;
}

extern "C" int64_t iss_resnet_workspace_bytes(const iss_resnet *net, int n_windows, int win_len)
{
    if (!net || n_windows < 0 || win_len < 1) return -1;
    const int64_t B = std::min(std::max(n_windows, 1), RES_BATCH);
    const int64_t act = max_act_per_window(net, win_len, nullptr);
    int64_t bytes = 0;
    bytes += 5 * (int64_t)align_up((size_t)B * act * 4, 256);
    bytes += align_up((size_t)B * net->feat_dim * win_len * 4, 256);
    bytes += align_up((size_t)B * 2 * net->c_final * net->h_final * 4, 256);
    bytes += align_up((size_t)(n_windows + 1) * 4, 256);
    return bytes;
}

extern "C" int iss_resnet_embed(iss_ctx *ctx, iss_resnet *net, const float *d_fea, int64_t M,
                                const int32_t *h_win_start, int n_windows, int win_len, float *d_emb,
                                void *d_work, int64_t work_bytes, void *stream)
{
    ISS_REQUIRE(ctx && net, ISS_ERR_INVALID, "iss_resnet_embed: NULL handle");
    if (n_windows <= 0) return ISS_OK;
    ISS_REQUIRE(d_fea && h_win_start && d_emb && d_work, ISS_ERR_INVALID, "iss_resnet_embed: NULL buffer");
    ISS_REQUIRE(win_len >= 1, ISS_ERR_INVALID, "iss_resnet_embed: win_len=%d", win_len);
    for (int i = 0; i < n_windows; ++i)
        ISS_REQUIRE(h_win_start[i] >= 0 && (int64_t)h_win_start[i] + win_len <= M, ISS_ERR_INVALID,
                    "iss_resnet_embed: window %d = [%d, %d) outside [0, %lld)", i, h_win_start[i], h_win_start[i] + win_len, (long long)M);
    ISS_REQUIRE(work_bytes >= iss_resnet_workspace_bytes(net, n_windows, win_len), ISS_ERR_INVALID,
                "iss_resnet_embed: workspace %lld < required %lld", (long long)work_bytes,
                (long long)iss_resnet_workspace_bytes(net, n_windows, win_len));
    ISS_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = iss_stream(stream);
    const int F = net->feat_dim, T = win_len;
    const int64_t B = std::min(n_windows, RES_BATCH);
    const int64_t act = max_act_per_window(net, T, nullptr);
    uint8_t *p = reinterpret_cast<uint8_t *>(d_work);
    size_t o = 0;
    float *buf[5];
    for (int i = 0; i < 5; ++i) { buf[i] = reinterpret_cast<float *>(p + o); o += align_up((size_t)B * act * 4, 256); }
    float *in0 = reinterpret_cast<float *>(p + o); o += align_up((size_t)B * F * T * 4, 256);
    float *pooled = reinterpret_cast<float *>(p + o); o += align_up((size_t)B * 2 * net->c_final * net->h_final * 4, 256);
    int32_t *d_start = reinterpret_cast<int32_t *>(p + o);
    ISS_CUDA_OK(cudaMemcpyAsync(d_start, h_win_start, sizeof(int32_t) * n_windows, cudaMemcpyHostToDevice, st));
    const float *blob = net->d_blob;

    // the filter shape and weights of a convolution (the batch, the spatial dims and the tensors are set per launch)
    auto conv_args = [&](const RConv &c) {
        ConvArgs a = {};
        a.w = blob + c.w_off; a.pre_scale = blob + c.scale_off; a.pre_shift = blob + c.shift_off;
        a.wt = c.wt;
        a.N = c.cout; a.K = c.kh * c.kw * c.cin; a.C = c.cin;
        a.KH = c.kh; a.KW = c.kw; a.SH = c.stride; a.SW = c.stride; a.PT = c.pad; a.PL = c.pad;
        a.flags = ISS_F_AFFINE_PRE;
        return a;
    };
    // Activation formats (conv_gemm.cuh): a tensor is stored as split-half words when its producer AND every consumer run on
    // engine 3 (every convolution of stages 2-4), fp32 otherwise.  Which engine runs a convolution does not depend on its
    // spatial dims, so this asks the kernel choice of the filter shape alone.
    const int mode = iss_get_gemm_mode();
    auto f16 = [&](const RConv &c) { return iss_conv_is_f16(iss_conv_kernel(conv_args(c), mode)); };
    auto conv = [&](const RConv &c, const float *in, bool in_packed, float *out, bool out_packed, int nb, int h, int w, int oh, int ow,
                    int flags, const float *residual, bool residual_packed) -> int {
        ConvArgs a = conv_args(c);
        a.in = in; a.residual = residual; a.out = out;
        a.in_packed = in_packed; a.out_packed = out_packed; a.residual_packed = residual_packed;
        a.M = (int64_t)nb * oh * ow; a.H = h; a.W = w; a.OH = oh; a.OW = ow;
        a.flags |= flags | (residual ? ISS_F_RESIDUAL : 0);
        return iss_launch_conv(a, mode, st);
    };

    for (int w0 = 0; w0 < n_windows; w0 += (int)B) {
        const int nb = std::min<int>((int)B, n_windows - w0);
        const int64_t tot = (int64_t)nb * F * T;
        window_gather_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(d_fea, d_start + w0, nb, T, F, in0);
        ISS_CUDA_OK(cudaGetLastError());
        iss_count_launch();
        int h = F, w = T;
        float *X = buf[0], *Y = buf[1], *A = buf[2], *Bf = buf[3], *S = buf[4];
        int rc = conv(net->stem, in0, false, X, false, nb, h, w, h, w, ISS_F_RELU, nullptr, false);
        if (rc != ISS_OK) return rc;
        bool x_packed = false;                                   // format of the block input X
        for (size_t bi = 0; bi < net->blocks.size(); ++bi) {
            const RBlock &b = net->blocks[bi];
            const int s = b.c2.stride;
            const int h2 = out_dim(h, 3, s, 1), w2 = out_dim(w, 3, s, 1);
            const bool a_packed = f16(b.c1) && f16(b.c2);        // c1 -> c2
            const bool b_packed = f16(b.c2) && f16(b.c3);        // c2 -> c3
            const bool s_packed = b.has_sc && f16(b.sc) && f16(b.c3);          // shortcut -> residual of c3
            bool y_packed = false;                               // c3 -> next block (its c1, its shortcut conv, the residual of its c3)
            if (bi + 1 < net->blocks.size()) {
                const RBlock &nx = net->blocks[bi + 1];
                y_packed = f16(b.c3) && f16(nx.c1) && f16(nx.c3) && (!nx.has_sc || f16(nx.sc));
            }
            rc = conv(b.c1, X, x_packed, A, a_packed, nb, h, w, h, w, ISS_F_RELU, nullptr, false);          if (rc != ISS_OK) return rc;
            rc = conv(b.c2, A, a_packed, Bf, b_packed, nb, h, w, h2, w2, ISS_F_RELU, nullptr, false);       if (rc != ISS_OK) return rc;
            const float *res = X;
            bool res_packed = x_packed;
            if (b.has_sc) {
                rc = conv(b.sc, X, x_packed, S, s_packed, nb, h, w, h2, w2, 0, nullptr, false);             if (rc != ISS_OK) return rc;
                res = S; res_packed = s_packed;
            }
            rc = conv(b.c3, Bf, b_packed, Y, y_packed, nb, h2, w2, h2, w2, ISS_F_RELU, res, res_packed);    if (rc != ISS_OK) return rc;
            std::swap(X, Y);
            x_packed = y_packed;
            h = h2; w = w2;
        }
        const int64_t np = (int64_t)nb * h * net->c_final;
        stat_pool_kernel<<<(unsigned)((np + 255) / 256), 256, 0, st>>>(X, nb, h, w, net->c_final, pooled);
        ISS_CUDA_OK(cudaGetLastError());
        iss_count_launch();
        ConvArgs a = {};
        a.in = pooled; a.w = blob + net->emb_w_off; a.bias = blob + net->emb_b_off; a.out = d_emb + (int64_t)w0 * net->embed_dim;
        a.M = nb; a.N = net->embed_dim; a.K = 2 * net->c_final * h;
        a.H = 1; a.W = 1; a.C = a.K; a.OH = 1; a.OW = 1; a.KH = 1; a.KW = 1; a.SH = 1; a.SW = 1;
        a.flags = ISS_F_BIAS;
        a.wt = net->emb_wt;
        rc = iss_launch_conv(a, mode, st);
        if (rc != ISS_OK) return rc;
    }
    return ISS_OK;
}
