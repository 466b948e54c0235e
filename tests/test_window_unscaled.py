"""CPU tests of unscaled records in a keyframe window (reprojection factors, item size (0, 0)): the host mirrors of
dfk_window_assemble (WindowBlocks.pack) and of the dense assembly (assemble_window) add such a record's residual b^T b to f
as it is and leave its inliers out of the inlier total; its blocks go where a photometric record's go."""
import numpy as np

from deepfactors_b200 import factors


def _records(rng, n, cs):
    npar = 12 + cs
    A = rng.standard_normal((n, 3 * npar, npar))
    JtJ = np.einsum("nki,nkj->nij", A, A).astype(np.float32)
    Jtr = rng.standard_normal((n, npar)).astype(np.float32)
    res = rng.uniform(1.0, 5.0, n).astype(np.float32)
    inl = rng.integers(10, 200, n)
    return JtJ, Jtr, res, inl


def test_pack_adds_unscaled_residuals_as_they_are_and_counts_photometric_inliers_only():
    cs = 8
    rng = np.random.default_rng(1)
    pairs = [(0, 1), (1, 0), (0, 2)]
    item_pair = [0, 0, 1, 1, 2]
    sizes = [(64, 48), (32, 24), (64, 48), (32, 24), (0, 0)]
    JtJ, Jtr, res, inl = _records(rng, len(item_pair), cs)
    lay = factors.WindowBlocks(3, cs, pairs)
    buf = lay.pack(item_pair, JtJ, Jtr, res, inl, sizes)
    o_t = lay.offsets()[2]
    f_photo = np.float32(0)
    for i in range(4):
        f_photo += np.float32(res[i]) / np.float32(inl[i]) * np.float32(sizes[i][0] * sizes[i][1])
    assert buf[o_t] == np.float32(f_photo + res[4])
    assert buf[o_t + 1] == float(inl[:4].sum())
    # without the unscaled record the photometric part is what it was
    ref = factors.WindowBlocks(3, cs, pairs).pack(item_pair[:4], JtJ[:4], Jtr[:4], res[:4], inl[:4], sizes[:4])
    assert ref[o_t] == f_photo and ref[o_t + 1] == buf[o_t + 1]
    # an unscaled record with no inliers still adds its residual (the pack of the photometric rule would skip it)
    inl0 = inl.copy()
    inl0[4] = 0
    assert lay.pack(item_pair, JtJ, Jtr, res, inl0, sizes)[o_t] == buf[o_t]


def test_dense_assembly_matches_block_buffer_with_a_link_only_keyframe():
    """keyframe 2 is tied to the window only by reprojection links (0 -> 2, 2 -> 0), as by a global loop closure"""
    cs = 8
    rng = np.random.default_rng(2)
    pairs = [(0, 1), (1, 0), (0, 2), (2, 0)]
    item_pair = [0, 0, 1, 1, 2, 3]
    sizes = [(64, 48), (32, 24), (64, 48), (32, 24), (0, 0), (0, 0)]
    JtJ, Jtr, res, inl = _records(rng, len(item_pair), cs)
    lay = factors.WindowBlocks(3, cs, pairs)
    buf = lay.pack(item_pair, JtJ, Jtr, res, inl, sizes)
    Hd, gd, f, ninl = lay.to_dense(buf)
    Hr, gr, fr = factors.assemble_window(factors.WindowLayout(3, cs), [pairs[p] for p in item_pair], JtJ, Jtr, res, inl,
                                         sizes)
    assert np.abs(Hd - Hr).max() <= 2e-6 * np.abs(Hr).max()
    assert np.abs(gd - gr).max() <= 2e-6 * np.abs(gr).max()
    assert abs(f - fr) <= 1e-6 * fr and ninl == float(inl[:4].sum())
    assert np.allclose(Hd, Hd.T)
    B = 6 + cs
    kf2 = slice(2 * B, 3 * B)
    assert np.abs(Hd[kf2, kf2]).max() > 0 and np.abs(Hd[0:B, kf2]).max() > 0   # the links reach keyframe 2
    assert not Hd[B:2 * B, kf2].any()                                         # keyframe 1 and 2 share no factor
    expect = sum(float(res[i]) / int(inl[i]) * sizes[i][0] * sizes[i][1] for i in range(4)) + float(res[4]) + float(res[5])
    assert abs(fr - expect) <= 1e-9 * expect


def test_unscaled_marker_is_both_sizes_zero():
    assert factors.is_unscaled((0, 0))
    assert not factors.is_unscaled((0, 5)) and not factors.is_unscaled((64, 48))
