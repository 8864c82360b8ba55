"""The online Viterbi decision rule (stream.online_step, the numpy model of iss_viterbi_online) against the offline
oracle: at every call the decided states are a prefix of the offline states, and after the end they are all of them."""
import numpy as np
import pytest

from oracle import viterbi_oracle as vo
from inaspeechsegmenter_b200.stream import computable_patches
from stream_oracle import online_step
from inaspeechsegmenter_b200 import pack


def _run_online(emis, trans, cuts):
    K = trans.shape[0]
    prior = np.log(np.ones(K) / K)[0]
    ref = vo.viterbi_numpy(emis, trans).astype(np.uint8)
    V, hist, got = None, np.zeros((0, K), dtype=np.int64), []
    bounds = [0] + sorted(cuts) + [len(emis)]
    for i, (a, b) in enumerate(zip(bounds[:-1], bounds[1:])):
        end = i == len(bounds) - 2
        dec, V, hist = online_step(emis[a:b], trans, prior, V, hist, a == 0, end)
        got.extend(dec.tolist())
        assert np.array_equal(np.array(got, dtype=np.uint8), ref[:len(got)]), (a, b)
        assert len(got) + len(hist) == b
    assert np.array_equal(np.array(got, dtype=np.uint8), ref)


@pytest.mark.parametrize('K,arg', [(2, 80), (3, 80), (2, 150), (3, 1)])
@pytest.mark.parametrize('seed', range(4))
def test_cnn_chains_random_splits(K, arg, seed):
    rng = np.random.default_rng(seed * 10 + K)
    T = int(rng.integers(1, 400))
    p = rng.dirichlet(np.ones(K) * 0.3, size=T).astype(np.float32)
    with np.errstate(divide='ignore'):
        emis = np.log(p).astype(np.float64)
    trans = vo.diag_trans_exp(arg, K)
    cuts = sorted(set(rng.integers(1, T, size=int(rng.integers(0, 12))).tolist())) if T > 1 else []
    _run_online(emis, trans, cuts)
    _run_online(emis, trans, list(range(1, T)))            # one step per call


def test_energy_chain_with_threshold_and_long_lag():
    rng = np.random.default_rng(3)
    loge = rng.normal(0, 1, size=3000).astype(np.float32)
    loge[500:2500] = 0.0                                    # exactly at the threshold: long ambiguous run
    thr = np.float64(np.float32(0.0))
    emis = vo.pred2logemission(loge > thr)
    trans = vo.log_trans_exp(150, cost0=-5)
    _run_online(emis, trans, sorted(rng.integers(1, 3000, size=40).tolist()))
    _run_online(emis[:300], trans, list(range(1, 300)))


def test_exact_ties():
    K = 3
    emis = np.zeros((200, K))                               # every path scores the same: first-max tie breaks only
    _run_online(emis, vo.diag_trans_exp(80, K), [1, 2, 3, 50, 51, 199])
    emis[::7, 1] = -np.inf
    _run_online(emis, vo.diag_trans_exp(0, K), list(range(1, 200, 3)))


def test_computable_patches_matches_patch_rows():
    for F in (68, 69, 70, 100, 1001):
        n = computable_patches(F)
        # every computable patch's last frame exists, and the next one's does not
        assert pack.patch_row0(10 ** 6, n - 1) + 67 <= F - 1 < pack.patch_row0(10 ** 6, n) + 67
    assert computable_patches(67) == 0
