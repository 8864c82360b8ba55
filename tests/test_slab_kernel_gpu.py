"""The slab kernel (csrc/conv_gemm_tc.cu, conv_slab_kernel) on the GPU: the 5x4 64->64 layer of both segmenter CNNs,
with the first layer fused into its fill (LD_FIRST) and from the stand-alone first layer's split-half words (LD_PACKED).

The A operand of every tap is a 64-row window of the 128-byte-swizzled slab that starts at any row; the wgmma descriptor
addresses it with the start address alone and a matrix base offset of 0 -- the swizzle follows the shared-memory
address bits, as tests/test_slab_indexing.py models it.  A wrong window would give wrong values here, not a fault.

Checked against the fp32 oracle (1e-4), the 3xTF32 engine and the fp32 CUDA-core engine (2e-5 per patch), on ranges
whose tiles straddle patches and end in a partial tile, on a single patch, and on more than 8192 patches (several
batches); the fused and the un-fused first layer agree; two runs are bit-for-bit identical."""
import os

import numpy as np
import pytest

from test_gpu_parity import _oracle_probs

pytestmark = pytest.mark.gpu

torch = pytest.importorskip('torch')


@pytest.fixture(scope='module')
def rt():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from inaspeechsegmenter_b200 import _lib, engine
    return dict(ctx=engine.Context(0), lib=_lib, engine=engine)


def _forward(rt, net, dm, ranges, mode, fuse_first):
    lib = rt['lib'].load()
    prev_mode, prev_env = lib.iss_get_gemm_mode(), os.environ.get('ISS_B200_FUSE_FIRST')
    try:
        os.environ['ISS_B200_FUSE_FIRST'] = '1' if fuse_first else '0'
        rt['lib'].check(lib.iss_set_gemm_mode(mode), 'set mode')
        l0 = lib.iss_launch_count()
        out = net.forward(dm, ranges).cpu().numpy()
        return out, lib.iss_launch_count() - l0
    finally:
        lib.iss_set_gemm_mode(prev_mode)
        if prev_env is None:
            os.environ.pop('ISS_B200_FUSE_FIRST', None)
        else:
            os.environ['ISS_B200_FUSE_FIRST'] = prev_env


@pytest.mark.parametrize('which,nmel', [('smn', 21), ('gender', 24)])
def test_slab_kernel_vs_oracle_and_other_engines(rt, synth_models, which, nmel):
    cfg, w = synth_models[which]
    rng = np.random.default_rng(2026 + nmel)
    L = 17000                                                # 8500 patches: more than one 8192-patch batch
    mspec = (rng.standard_normal((L, 24)) * 3 - 5).astype(np.float32)
    P = (L + 1) // 2
    net = rt['engine'].CnnModel.from_keras(rt['ctx'], cfg, w, nmel)
    dm = torch.from_numpy(mspec).cuda()
    for ranges in ([(0, 1), (5, 612), (700, 1500)], [(37, 38)], [(0, P)]):
        ref = _oracle_probs(cfg, w, mspec, nmel, ranges)
        fused, n_fused = _forward(rt, net, dm, ranges, 3, True)
        again, _ = _forward(rt, net, dm, ranges, 3, True)
        plain, n_plain = _forward(rt, net, dm, ranges, 3, False)
        eng2, n_eng2 = _forward(rt, net, dm, ranges, 2, True)
        eng0, _ = _forward(rt, net, dm, ranges, 0, True)
        assert np.array_equal(fused, again)
        for name, got in (('fused', fused), ('unfused', plain)):
            assert np.abs(got - ref).max() <= 1e-4, (name, ranges[0])
            assert np.abs(got - eng2).max() <= 2e-5, (name, ranges[0])
            assert np.abs(got - eng0).max() <= 2e-5, (name, ranges[0])
        assert np.abs(fused - plain).max() <= 2e-5
        assert n_fused <= n_eng2 and n_plain <= n_eng2
