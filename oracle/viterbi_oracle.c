/* Oracle (test infrastructure): max-sum Viterbi decoding, plain C.
 *
 * CPU restatement of reference inaSpeechSegmenter/pyannote_viterbi.py:118-224
 * for the only way segmenter.py calls it (segmenter.py:72,176): no
 * `consecutive`, no `constraint`, no `initial` => the state-duplication
 * helpers (:51-115) are identities and the prior is log(1/K) (:166-167).
 *
 *   V[0,j]  = E[0,j] + log(1/K)                                   (:194)
 *   P[t,j]  = argmax_k ( V[t-1,k] + A[k,j] )   first max on ties   (:207-210)
 *   V[t,j]  = E[t,j] + ( V[t-1,P[t,j]] + A[P[t,j],j] )             (:213)
 *   X[T-1]  = argmax_j V[T-1,j] ; X[t-1] = P[t, X[t]]              (:217-220)
 *
 * All arithmetic in IEEE double, evaluated in exactly that order, so results
 * are bit-identical to numpy's.  NaN handling follows numpy.argmax: the first
 * NaN wins.  Built by oracle/Makefile into oracle/_build/liboracle.so; used by
 * tests and by bench.py's cpu_baseline leg only.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#define ORACLE_MAXK 8

static int argmax_first(const double *v, int n)
{
    /* numpy.argmax semantics: first maximum; a NaN is larger than anything. */
    int best = 0;
    double bv = v[0];
    if (isnan(bv)) return 0;
    for (int i = 1; i < n; ++i) {
        if (isnan(v[i])) return i;
        if (v[i] > bv) { bv = v[i]; best = i; }
    }
    return best;
}

/* A partial chain: the same DP on steps [0, T) of a longer chain, in the same order of double operations.
 *   vin       [K] scores V[-1] of the step before the first, or NULL.  With vin the first step is an ordinary
 *             transition from it; without, V[0] = E[0] + log(1/K).
 *   vout      [K] out: V[T-1] (or NULL).
 *   backmap   [K] out: for each end state x, the state the path ending in x has before the first step (with vin)
 *             or at the first step (without); NULL to skip.
 *   end_state -1: backtrack from the first argmax of V[T-1]; else from that state.
 *   states    out: X[t] for every t % out_stride == 0, at states[t / out_stride] (or NULL).
 * Returns 0 on success. */
int oracle_viterbi_partial(const double *emission, const double *trans, int64_t T, int K, const double *vin,
                           double *vout, int32_t *backmap, int end_state, int out_stride, int32_t *states)
{
    if (K < 1 || K > ORACLE_MAXK || T < 1 || out_stride < 1 || end_state < -1 || end_state >= K) return -1;
    uint8_t *bp = (uint8_t *)malloc((size_t)T * (size_t)K);
    if (!bp) return -2;
    double V[ORACLE_MAXK], Vn[ORACLE_MAXK], cand[ORACLE_MAXK];
    int64_t t = 0;
    if (!vin) {
        /* np.log(np.ones(k) / k) */
        const double prior = log(1.0 / (double)K);
        for (int j = 0; j < K; ++j) { V[j] = emission[j] + prior; bp[j] = (uint8_t)j; }
        t = 1;
    } else {
        for (int j = 0; j < K; ++j) V[j] = vin[j];
    }
    for (; t < T; ++t) {
        const double *e = emission + t * K;
        for (int j = 0; j < K; ++j) {
            for (int k = 0; k < K; ++k) cand[k] = V[k] + trans[k * K + j];
            int a = argmax_first(cand, K);
            bp[t * K + j] = (uint8_t)a;
            Vn[j] = e[j] + cand[a];
        }
        for (int j = 0; j < K; ++j) V[j] = Vn[j];
    }
    if (vout) for (int j = 0; j < K; ++j) vout[j] = V[j];
    if (backmap) {
        for (int x0 = 0; x0 < K; ++x0) {
            int x = x0;
            for (int64_t s = T - 1; s >= (vin ? 0 : 1); --s) x = bp[s * K + x];
            backmap[x0] = x;
        }
    }
    if (states) {
        int x = end_state >= 0 ? end_state : argmax_first(V, K);
        for (int64_t s = T - 1; s >= 0; --s) {
            if (s % out_stride == 0) states[s / out_stride] = x;
            if (s > 0) x = bp[s * K + x];
        }
    }
    free(bp);
    return 0;
}

/* emission: [T,K] row-major doubles; trans: [K,K] (from,to); states: [T] out.
 * scratch for back-pointers is allocated here. returns 0 on success. */
int oracle_viterbi(const double *emission, const double *trans, int64_t T, int K,
                   int32_t *states)
{
    return oracle_viterbi_partial(emission, trans, T, K, NULL, NULL, NULL, -1, 1, states);
}

/* float32 emissions (np.log(r) of a float32 softmax, segmenter.py:176):
 * numpy promotes float32 + float64 to float64 element-wise, i.e. each emission
 * is widened exactly before the add. */
int oracle_viterbi_f32(const float *emission, const double *trans, int64_t T, int K,
                       int32_t *states)
{
    double *e = (double *)malloc((size_t)T * (size_t)K * sizeof(double));
    if (!e) return -2;
    for (int64_t i = 0; i < T * K; ++i) e[i] = (double)emission[i];
    int rc = oracle_viterbi(e, trans, T, K, states);
    free(e);
    return rc;
}
