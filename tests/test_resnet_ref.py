"""CPU: the float64 evaluator of the x-vector extractor blob (oracle/resnet_ref.py) against the fp32 evaluations of the
same network -- vbx_oracle.ResNet101Oracle, the blob evaluator of test_onnx_reader and the outputs of the real resnet.py
stored in the goldens.  Their fp32 error must lie inside the bound the evaluator propagates for the fp32 engine (mode 0):
this pins the reference the GPU probes (test_resnet_probes_gpu.py) are checked against, without a GPU."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import resnet_ref as rr
from oracle import vbx_oracle as vx
from test_onnx_reader import _eval_blob

HERE = os.path.dirname(os.path.abspath(__file__))

# the probe architectures of test_resnet_probes_gpu.py: (m, feat_dim, num_blocks)
PROBE_ARCHS = [(32, 64, (1, 2, 1, 1)), (64, 64, (1, 1, 0, 0)), (16, 64, (2, 1, 1, 0)), (8, 64, (2, 1, 0, 0)),
               (32, 64, (0, 0, 0, 0)), (32, 40, (1, 1, 1, 1))]


def _within(got, ref, E, c=1.0):
    r = np.abs(np.asarray(got, dtype=np.float64) - ref) / E
    assert np.isfinite(r).all() and r.max() <= c, r.max()
    return float(r.max())


@pytest.mark.parametrize('m,feat,nb', PROBE_ARCHS)
def test_reference_matches_fp32_blob_evaluator_on_probe_archs(m, feat, nb):
    arch = rr.plan(m, feat, 32, nb)
    blob = rr.synthetic_blob(arch, seed=m + sum(nb))
    x = np.random.default_rng(1).standard_normal((3, feat, 144)).astype(np.float32)
    y, E = rr.forward(arch, blob, x, mode=0)
    got = _eval_blob(blob, m, feat, 32, nb, torch.from_numpy(x))
    _within(got, y, E)
    # a short (tail) window: odd widths into the stride-2 layers
    y, E = rr.forward(arch, blob, x[:1, :, :17], mode=0)
    _within(_eval_blob(blob, m, feat, 32, nb, torch.from_numpy(x[:1, :, :17])), y, E)


def test_reference_matches_resnet101_oracle_and_golden(golden):
    """The release architecture with the seeded weights: ResNet101Oracle (fp32) and the real resnet.py outputs
    (resnet_y: two 144-frame windows, resnet_ys: a 131-frame tail window) lie inside the mode-0 bound."""
    from inaspeechsegmenter_b200.vbx_segmenter import resnet_blob_from_state
    sd = vx.synthetic_resnet101_state(seed=5)
    arch = rr.plan(**rr.RELEASE)
    blob = resnet_blob_from_state(sd)
    assert blob.size == arch.blob_len
    x = golden['resnet_x'][:1]
    y, E = rr.forward(arch, blob, x, mode=0)
    _within(golden['resnet_y'][:1], y, E)
    _within(vx.ResNet101Oracle(sd, threads=4).forward(torch.from_numpy(x)).numpy(), y, E)
    ys, Es = rr.forward(arch, blob, golden['resnet_xs'], mode=0)
    _within(golden['resnet_ys'], ys, Es)
    # the bound is a scale of fp32 round-off, not a blanket tolerance: 1e-4 max|y| is far above it
    assert E.max() < 2e-5 * np.abs(y).max()


def test_reference_matches_real_module_small():
    """tests/golden/resnet_small.npz: the real resnet.py module (m = 4, blocks (2, 1, 1, 1), feat 16, embed 8)."""
    from inaspeechsegmenter_b200.vbx_segmenter import resnet_blob_from_state
    z = np.load(os.path.join(HERE, 'golden', 'resnet_small.npz'))
    sd = {k[3:]: z[k] for k in z.files if k.startswith('sd:')}
    arch = rr.plan(4, 16, 8, (2, 1, 1, 1))
    blob = resnet_blob_from_state(sd, m=4, num_blocks=(2, 1, 1, 1))
    assert blob.size == arch.blob_len
    y, E = rr.forward(arch, blob, z['x'], mode=0)
    _within(z['y'], y, E)


def test_plan_matches_library_blob_length():
    """The architecture walk agrees with build_plan (iss_resnet_blob_len of the library, when it is built)."""
    from inaspeechsegmenter_b200 import _lib
    try:
        lib = _lib.load(build_if_missing=False)
    except (OSError, _lib.IssError):
        pytest.skip('libiss_b200.so not built')
    for m, feat, nb in PROBE_ARCHS + [(32, 64, (3, 4, 23, 3)), (4, 16, (2, 1, 1, 1))]:
        a = (ctypes.c_int * 4)(*nb)
        assert rr.plan(m, feat, 32, nb).blob_len == lib.iss_resnet_blob_len(m, feat, 32, ctypes.cast(a, ctypes.c_void_p))


def _conv(k, stride, cin, cout, images='f16'):
    return dict(k=k, stride=stride, pad=1 if k == 3 else 0, cin=cin, cout=cout, images=images)


def test_dispatch_follows_the_kernel_selector_rules():
    """conv_kernel against the rules of iss_conv_kernel / iss_prepare_weights (conv_gemm.cuh): engine 2 takes C, K and N
    multiples of 32; engine 3 (mode 3 only) C and N multiples of 64; the small-N kernel 1x1 stride-1 layers with N <= 8
    and no residual in every mode; the stem has no tensor-core images; mode 0 is fp32 throughout."""
    for k in (1, 3):
        for stride in (1, 2):
            for cin in (8, 16, 32, 48, 64, 96, 128, 256):
                for cout in (8, 16, 32, 64, 96, 128, 512):
                    c = _conv(k, stride, cin, cout)
                    small = k == 1 and stride == 1 and cout <= 8 and cin * cout * 4 <= 48 * 1024
                    e2 = cin % 32 == 0 and cout % 32 == 0
                    e3 = e2 and cin % 64 == 0 and cout % 64 == 0
                    for mode in (0, 2, 3):
                        got = rr.conv_kernel(c, mode)
                        if small:
                            assert got == rr.K_SMALL_N
                            assert rr.conv_kernel(c, mode, residual=True) != rr.K_SMALL_N
                        elif mode == 0 or not e2:
                            assert got == rr.K_F32, (c, mode)
                        elif mode == 3 and e3:
                            slab = k == 1 and stride == 1 and cin == 64 and cout == 64
                            assert got == (rr.K_SLAB if slab else rr.K_F16), (c, mode)
                        else:
                            assert got == rr.K_TF32, (c, mode)
                        assert rr.unit_error(got) == (rr.U_SPLIT if got in (rr.K_TF32, rr.K_F16, rr.K_SLAB) else rr.U32)
    for m in (8, 16, 32, 64, 128):
        arch = rr.plan(m, 64, 32, (1, 1, 1, 1))
        for mode in (0, 2, 3):
            assert rr.conv_kernel(arch.stem, mode) == rr.K_F32
        assert rr.conv_kernel(arch.emb, 2) == rr.conv_kernel(arch.emb, 3) == rr.K_TF32   # no fp16 image
        assert rr.conv_kernel(arch.emb, 0) == rr.K_F32


def test_release_formats():
    """The release network on the default engine: stage 1 on engine 2 with fp32 tensors, stages 2-4 on engine 3 with
    split-half words between their layers; the stage-2 entry reads the fp32 stage-1 output."""
    arch = rr.plan(**rr.RELEASE)
    fm = rr.packed_formats(arch, 3)
    st = [int(b['name'][5]) for b in arch.blocks]
    for b, f, s in zip(arch.blocks, fm, st):
        engine = rr.K_TF32 if s == 1 else rr.K_F16
        assert all(rr.conv_kernel(b[c], 3) == engine for c in ('c1', 'c2', 'c3') if b[c] is not None)
        assert f['a'] == f['b'] == (s > 1)
        assert f['s'] == (s > 1 and b['sc'] is not None)
    assert [f['y'] for f in fm] == [False] * 3 + [True] * (len(fm) - 4) + [False]
    names = rr.kernel_names(arch, 3)
    assert 'conv_gemm_wg_kernel<1,64,0>' in names and 'conv_gemm_wg_kernel<1,128,1>' in names
    assert not any('slab' in n or 'small_n' in n for n in names)


def test_stat_pool_bound_is_finite_on_constant_channels():
    """A constant channel: the float64 std is exactly sqrt(1e-10) and its bound finite (sqrt(E_var), not E_var / 2 std)."""
    x = torch.full((1, 2, 3, 144), 0.7, dtype=torch.float64)
    p, Ep = rr.stat_pool(x, torch.zeros_like(x))
    assert torch.equal(p[0, 6:], torch.full((6,), 1e-5, dtype=torch.float64))
    assert torch.isfinite(Ep).all() and (Ep[0, 6:] < 1e-2).all()
