// mlp.cu -- stack of Dense layers (the gender-detection MLP applied to x-vectors by
// VoiceFemininityScoring, inaSpeechSegmenter/vbx_segmenter.py:116-124,188-191: a Keras
// Sequential loaded from interspeech2023_{all,cvfr}.hdf5 and run with model.predict).
// Each layer is one launch of the shared implicit-GEMM (conv_gemm.cu, fp32 CUDA cores: the
// matrices are [n_windows x 256] -- tiny) with the fused bias / BatchNorm-affine / ReLU / sigmoid epilogue.
#include <vector>

#include "conv_gemm.cuh"

struct iss_mlp {
    iss_ctx *ctx;
    std::vector<iss_layer_desc> layers;
    float *d_blob;
    int in_dim, out_dim, max_dim;
};

extern "C" int iss_mlp_create(iss_ctx *ctx, const iss_layer_desc *layers, int n_layers, const float *h_blob,
                              int64_t blob_len, int in_dim, iss_mlp **out)
{
    ISS_REQUIRE(ctx && layers && h_blob && out && n_layers > 0 && in_dim > 0, ISS_ERR_INVALID, "iss_mlp_create: bad argument");
    ISS_CUDA_OK(cudaSetDevice(ctx->device));
    iss_mlp *m = new iss_mlp();
    m->ctx = ctx; m->d_blob = nullptr; m->in_dim = in_dim;
    int dim = in_dim, mx = in_dim;
    auto ok_off = [&](int64_t off, int64_t len) { return off >= 0 && off + len <= blob_len; };
    for (int i = 0; i < n_layers; ++i) {
        const iss_layer_desc &d = layers[i];
        bool ok = d.kind == ISS_LAYER_DENSE && d.cin == dim && d.cout >= 1 && ok_off(d.w_off, (int64_t)d.cin * d.cout) &&
                  !(d.flags & ISS_F_SOFTMAX);
        if (ok && (d.flags & ISS_F_BIAS)) ok = ok_off(d.bias_off, d.cout);
        if (ok && (d.flags & ISS_F_AFFINE_PRE)) ok = ok_off(d.pre_scale_off, d.cout) && ok_off(d.pre_shift_off, d.cout);
        if (ok && (d.flags & ISS_F_AFFINE_POST)) ok = ok_off(d.post_scale_off, d.cout) && ok_off(d.post_shift_off, d.cout);
        if (!ok) { delete m; iss_set_error("iss_mlp_create: layer %d is not a Dense layer consistent with input width %d", i, dim); return ISS_ERR_UNSUPPORTED; }
        m->layers.push_back(d);
        dim = d.cout;
        mx = dim > mx ? dim : mx;
    }
    m->out_dim = dim; m->max_dim = mx;
    cudaError_t e = cudaMalloc(&m->d_blob, (size_t)blob_len * sizeof(float));
    if (e != cudaSuccess) { delete m; iss_set_error("cudaMalloc mlp blob: %s", cudaGetErrorString(e)); return ISS_ERR_NOMEM; }
    e = cudaMemcpy(m->d_blob, h_blob, (size_t)blob_len * sizeof(float), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) { cudaFree(m->d_blob); delete m; iss_set_error("cudaMemcpy mlp blob: %s", cudaGetErrorString(e)); return ISS_ERR_CUDA; }
    *out = m;
    return ISS_OK;
}

extern "C" int iss_mlp_destroy(iss_mlp *m)
{
    if (!m) return ISS_OK;
    cudaSetDevice(m->ctx->device);
    if (m->d_blob) cudaFree(m->d_blob);
    delete m;
    return ISS_OK;
}

extern "C" int iss_mlp_out_dim(const iss_mlp *m) { return m ? m->out_dim : -1; }

extern "C" int64_t iss_mlp_workspace_bytes(const iss_mlp *m, int64_t n_rows)
{
    if (!m || n_rows < 0) return -1;
    return 2 * ((n_rows * m->max_dim * 4 + 255) / 256 * 256) + 256;
}

extern "C" int iss_mlp_forward(iss_ctx *ctx, iss_mlp *m, const float *d_x, int64_t n_rows, float *d_y,
                               void *d_work, int64_t work_bytes, void *stream)
{
    ISS_REQUIRE(ctx && m, ISS_ERR_INVALID, "iss_mlp_forward: NULL handle");
    if (n_rows <= 0) return ISS_OK;
    ISS_REQUIRE(d_x && d_y && d_work && work_bytes >= iss_mlp_workspace_bytes(m, n_rows), ISS_ERR_INVALID, "iss_mlp_forward: bad buffer");
    // the fp32 kernels read rows with float4 loads (conv_gemm_f32_kernel when C % 8 == 0, dense_small_n_kernel when
    // K % 4 == 0) and store them with float4 stores, without checking the base pointers
    ISS_REQUIRE(((uintptr_t)d_x | (uintptr_t)d_y | (uintptr_t)d_work) % 16 == 0, ISS_ERR_INVALID,
                "iss_mlp_forward: d_x, d_y and d_work must be 16-byte aligned");
    ISS_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = iss_stream(stream);
    const size_t half = (size_t)((n_rows * m->max_dim * 4 + 255) / 256 * 256);
    float *buf[2] = {reinterpret_cast<float *>(d_work), reinterpret_cast<float *>(reinterpret_cast<unsigned char *>(d_work) + half)};
    const float *cur = d_x;
    for (size_t i = 0; i < m->layers.size(); ++i) {
        const iss_layer_desc &d = m->layers[i];
        ConvArgs a = {};
        a.in = cur; a.w = m->d_blob + d.w_off;
        a.bias = (d.flags & ISS_F_BIAS) ? m->d_blob + d.bias_off : nullptr;
        a.pre_scale = (d.flags & ISS_F_AFFINE_PRE) ? m->d_blob + d.pre_scale_off : nullptr;
        a.pre_shift = (d.flags & ISS_F_AFFINE_PRE) ? m->d_blob + d.pre_shift_off : nullptr;
        a.post_scale = (d.flags & ISS_F_AFFINE_POST) ? m->d_blob + d.post_scale_off : nullptr;
        a.post_shift = (d.flags & ISS_F_AFFINE_POST) ? m->d_blob + d.post_shift_off : nullptr;
        a.out = (i + 1 == m->layers.size()) ? d_y : buf[i & 1];
        a.M = n_rows; a.N = d.cout; a.K = d.cin; a.H = 1; a.W = 1; a.C = d.cin; a.OH = 1; a.OW = 1;
        a.KH = 1; a.KW = 1; a.SH = 1; a.SW = 1; a.flags = d.flags;
        int rc = iss_launch_conv(a, ISS_GEMM_FP32, st);
        if (rc != ISS_OK) return rc;
        cur = a.out;
    }
    return ISS_OK;
}
