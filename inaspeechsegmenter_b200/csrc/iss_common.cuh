// iss_common.cuh -- shared declarations of libiss_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

#include "../../include/iss_b200.h"

void iss_set_error(const char *fmt, ...);
void iss_count_launch(int n = 1);
// cudaFuncAttributeMaxDynamicSharedMemorySize is per device: opts `func` in once per (kernel, current device)
cudaError_t iss_optin_smem(const void *func, int bytes);

#define ISS_CUDA_OK(call)                                                              \
    do {                                                                               \
        cudaError_t _e = (call);                                                       \
        if (_e != cudaSuccess) {                                                       \
            iss_set_error("%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e)); \
            return ISS_ERR_CUDA;                                                       \
        }                                                                              \
    } while (0)

#define ISS_REQUIRE(cond, code, ...)                                                   \
    do {                                                                               \
        if (!(cond)) { iss_set_error(__VA_ARGS__); return (code); }                    \
    } while (0)

// ---- sidekit front-end constants (sidekit_mfcc.py:214-220, segmenter.py:58) ----
constexpr int ISS_WIN = 400;
constexpr int ISS_HOP = 160;
constexpr int ISS_NFFT = 512;
constexpr int ISS_NBIN = 257;
constexpr int ISS_NMEL = 24;
constexpr int ISS_FB_MAXNNZ = 512;     // trfbank(16000,512,100,8000,0,24) has 454 non-zeros

struct SidekitTables {
    // sparse mel filterbank: filter m covers bins [lo[m], lo[m]+cnt[m]) with weights w[off[m]..]
    int lo[ISS_NMEL];
    int cnt[ISS_NMEL];
    int off[ISS_NMEL];
    int nnz;
    float w[ISS_FB_MAXNNZ];
    // the same sums as <= 32 balanced tasks (one per lane): task t covers bins [task_lo, task_lo + task_cnt) with weights
    // w[task_off ..]; filter m is the sum of tasks [filt_first[m], filt_first[m] + filt_n[m]) (feat_sidekit.cu)
    int task_lo[32], task_cnt[32], task_off[32];
    int filt_first[ISS_NMEL], filt_n[ISS_NMEL];
    float win32[ISS_WIN];
    double win64[ISS_WIN];
    float tw256_32[2 * 256];   // W_256^m  (cos, -sin) interleaved
    double tw256_64[2 * 256];
    float tw512_32[2 * 257];   // W_512^k, k = 0..256
    double tw512_64[2 * 257];
};

struct iss_ctx {
    int device;
    int sm_count;
    SidekitTables *d_tables;     // device copy
    bool tables_ready;
    double *d_partials;          // per-tile {sum, count} partials of loge
    int64_t partials_cap;        // in tiles
    void *d_recs;                // per-recording table of a features call (feat_sidekit.cu)
    int64_t recs_cap;            // in entries
    void *d_vbx_recs;            // record table of a VBx features or dither call (feat_vbx.cu)
    int64_t vbx_recs_cap;        // in bytes
    void *resample;              // tap tables and recording table of the resampler (resample.cu)
};

// Frees the resampler's device memory of a context (resample.cu).
void iss_resample_free(iss_ctx *ctx);

static inline cudaStream_t iss_stream(void *s) { return reinterpret_cast<cudaStream_t>(s); }
