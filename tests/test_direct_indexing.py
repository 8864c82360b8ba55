"""CPU model of the addressing of the wgmma convolution kernel (csrc/conv_gemm_tc.cu, conv_gemm_wg_kernel).

The kernel cannot run here; its index arithmetic can.  A CTA owns GEMM rows m0 .. m0 + 127, warpgroup g rows
m0 + 64 g ..; thread t of a warpgroup fills rows t // 8 + 16 i (i < 4), 16-byte chunk j = t % 8 of the 128-byte operand
row of each k-block, at chunk j ^ (row & 7) of the SWIZZLE_128B tile (row_dst0).  The k-blocks walk the taps as
k = (rr * KW + ss) * C + c0; taps outside the input are zero.  wgmma reads logical element k of row r from chunk
(k // EPC) ^ (r & 7).  The fp32 accumulator register q of thread t holds row 16 (t // 32) + (t % 32) // 4 + 8 ((q % 4) // 2),
column 8 (q // 4) + 2 (t % 4) + q % 2, which the epilogue stores at out[m][n].  Checked against the definition of a
convolution for both engines (64 fp16 / 32 TF32 values per operand row), stride 1 and 'same' padding, including the
zero-filled tail of the last tile."""
import numpy as np
import pytest

TBM = 128


def kernel_conv(x, w, SH, SW, PT, PL, OH, OW, KE, BN=64):
    """x [n, H, W, C], w [KH, KW, C, N] (float64) -> y [n, OH, OW, N] through the kernel's fill, read and epilogue."""
    n, H, W, C = x.shape
    KH, KW, _, N = w.shape
    assert C % KE == 0 and N % BN == 0
    EPC = KE // 8                                            # values per 16-byte chunk of the operand row
    M, K = n * OH * OW, KH * KW * C
    nkb = K // KE
    flat = x.reshape(-1)
    wt = w.reshape(K, N)
    gm = (M + TBM - 1) // TBM
    out = np.full((M, N), np.nan)
    t = np.arange(128)
    j = t & 7
    for bx in range(gm):
        for g in range(2):
            m0 = bx * TBM + g * 64
            rows = (t[:, None] >> 3) + 16 * np.arange(4)[None, :]          # [t, i] local row
            m = m0 + rows
            ok_row = m < M
            mm = np.where(ok_row, m, 0)
            img, rem = mm // (OH * OW), mm % (OH * OW)
            ih0, iw0 = (rem // OW) * SH - PT, (rem % OW) * SW - PL
            row_dst = np.broadcast_to((t[:, None] >> 3) & 7, rows.shape)     # row_dst0: (t / 8 + 16 i) & 7 == (t / 8) & 7
            assert np.array_equal(row_dst, rows & 7)
            A = np.zeros((64, K))
            c0 = ss = rr = 0
            for kb in range(nkb):
                tile = np.zeros((64, 8, EPC))                                # the swizzled operand tile of this k-block
                ih, iw = ih0 + rr, iw0 + ss
                ok = ok_row & (ih >= 0) & (ih < H) & (iw >= 0) & (iw < W)
                base = ((img * H + ih) * W + iw) * C + c0 + j[:, None] * EPC
                vals = np.where(ok[..., None], flat[np.where(ok, base, 0)[..., None] + np.arange(EPC)], 0.0)
                tile[rows, j[:, None] ^ row_dst] = vals
                # wgmma's view: element k of row r at chunk (k // EPC) ^ (r & 7)
                r = np.arange(64)[:, None]
                k = np.arange(KE)[None, :]
                A[:, kb * KE:(kb + 1) * KE] = tile[r, (k // EPC) ^ (r & 7), k % EPC]
                c0 += KE
                if c0 == C:
                    c0 = 0
                    ss += 1
                    if ss == KW:
                        ss, rr = 0, rr + 1
            for nt in range(N // BN):
                D = A @ wt[:, nt * BN:(nt + 1) * BN]                        # [64, BN], the warpgroup's accumulator tile
                q = np.arange(BN // 2)
                wq, lq = t[:, None] >> 5, t[:, None] & 31
                dr = 16 * wq + (lq >> 2) + 8 * ((q[None, :] & 3) >> 1)
                dc = 8 * (q[None, :] >> 2) + 2 * (lq & 3) + (q[None, :] & 1)
                assert len(set(zip(dr.ravel().tolist(), dc.ravel().tolist()))) == 64 * BN    # every element exactly once
                live = m0 + dr < M
                out[(m0 + dr)[live], (nt * BN + dc)[live]] = D[dr, dc][live]
    return out.reshape(n, OH, OW, N)


def reference_conv(x, w, SH, SW, PT, PL, OH, OW):
    n, H, W, C = x.shape
    KH, KW, _, N = w.shape
    xp = np.zeros((n, max(H + PT, (OH - 1) * SH + KH), max(W + PL, (OW - 1) * SW + KW), C))
    xp[:, PT:PT + H, PL:PL + W] = x
    y = np.zeros((n, OH, OW, N))
    for a in range(KH):
        for b in range(KW):
            y += np.einsum('nhwc,cd->nhwd', xp[:, a:a + (OH - 1) * SH + 1:SH, b:b + (OW - 1) * SW + 1:SW], w[a, b])
    return y


@pytest.mark.parametrize('n,H,W,KH,KW', [(3, 65, 17, 5, 4), (5, 9, 7, 3, 3), (2, 30, 7, 3, 3), (7, 6, 5, 2, 4), (1, 65, 20, 5, 4)])
def test_direct_addressing_is_a_valid_convolution(n, H, W, KH, KW):
    rng = np.random.default_rng(n * 1000 + H)
    for C, KE in ((64, 64), (32, 32)):                          # engine 3 (fp16 split) / engine 2 (3xTF32)
        x = rng.standard_normal((n, H, W, C))
        w = rng.standard_normal((KH, KW, C, 64))
        OH, OW = H - KH + 1, W - KW + 1
        y = kernel_conv(x, w, 1, 1, 0, 0, OH, OW, KE)
        np.testing.assert_allclose(y, reference_conv(x, w, 1, 1, 0, 0, OH, OW), rtol=1e-12, atol=1e-10)


def test_useful_row_fraction_of_the_segmenter_layer():
    """The 128-row tiles run over the whole batch (rows of consecutive patches share a tile), so only the last tile of a
    launch carries idle rows: for the dominant segmenter layer (65 x 17 input, 5 x 4 filter) at the 8192-patch batch
    fewer than one GEMM row in 10 000 is idle."""
    H, W, KH, KW, B = 65, 17, 5, 4, 8192
    M = B * (H - KH + 1) * (W - KW + 1)
    tiles = (M + TBM - 1) // TBM
    assert M / (tiles * TBM) > 0.9999


@pytest.mark.parametrize('n,H,W', [(3, 16, 36), (5, 8, 18), (2, 5, 3), (1, 1, 1), (4, 7, 40)])
def test_padded_direct_addressing_is_a_same_convolution(n, H, W):
    """'same' 3x3 convolutions (ResNet101) with stride 1 and 2: padding by the bounds check of the fill."""
    rng = np.random.default_rng(n * 100 + W)
    for S in (1, 2):
        x = rng.standard_normal((n, H, W, 64))
        w = rng.standard_normal((3, 3, 64, 128))
        OH, OW = (H - 1) // S + 1, (W - 1) // S + 1
        y = kernel_conv(x, w, S, S, 1, 1, OH, OW, 64, BN=128)
        np.testing.assert_allclose(y, reference_conv(x, w, S, S, 1, 1, OH, OW), rtol=1e-12, atol=1e-10)
