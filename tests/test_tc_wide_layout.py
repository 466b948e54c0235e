"""CPU model of the tensor-core partial of the wide code sizes (dfk_sfm_tc_wide.cu, TcCfg in dfk_internal.h).

  * the operand packing A = [code-l 0..S-1 ; h 0..F-1], B = [h 0..F-1 ; code-l S..C-1 ; pose-l], S = C - 8, and the
    index map the finalize reads (hh / lh) rebuild HH + LH + LH^T of the reduced rows exactly, at C = 32, 64 and 128;
  * what the kernel writes of D (neither the l*l block nor the lower triangle of HH) covers every entry the finalize
    reads;
  * on the inputs of the GPU tests, the split-tf32 sum passes the per-entry bars by a factor of 50 at C = 64 and 128,
    and the comparator rejects the two packing bugs that matter at C = 128 (the l rows of the features kept in B lost,
    LH^T missing) by a factor of 4.
"""
import numpy as np
import pytest

from oracle import oracle as orc
from system_accuracy import H_BAR, JTR_BAR, assert_system_close, case_pair, level_reference
from test_system_accuracy import _rejected, emulated_gram, gram_result, tf32_split, valid_rows


@pytest.fixture(scope="module", autouse=True)
def _built_oracle():
    orc.build()


class Layout:
    """TcCfg<C>: D = A B^T (ROWS x COLS) stored column-major"""

    def __init__(self, C):
        self.C, self.S, self.F = C, C - 8, C + 8
        self.ROWS, self.COLS = 2 * C, C + 24
        self.a_rows = [("l", f) for f in range(self.S)] + [("h", f) for f in range(self.F)]
        self.b_cols = [("h", f) for f in range(self.F)] + [("l", f) for f in range(self.S, self.F)]
        assert len(self.a_rows) == self.ROWS and len(self.b_cols) == self.COLS

    def hh(self, i, j):
        return j * self.ROWS + self.S + i

    def lh(self, i, j):
        return j * self.ROWS + i if i < self.S else (16 + i) * self.ROWS + self.S + j

    def written(self, m, n):
        """the kernel's flush condition"""
        return n < self.F if m < self.S else (n >= self.F or n >= m - self.S)

    def d_of(self, h, l):
        """D of the rows h, l (pixels x F), products summed in fp64"""
        val = {"h": h, "l": l}
        A = np.stack([val[k][:, f] for k, f in self.a_rows], 1)
        B = np.stack([val[k][:, f] for k, f in self.b_cols], 1)
        return (A.T @ B).T.reshape(-1)  # column-major

    def finalize_reads(self):
        """(i, j) pairs, i <= j, the finalize kernel reads: code rows u (columns u .. C+6) and the 7x7 pose block"""
        C = self.C
        pairs = [(u, j) for u in range(C) for j in range(u, C + 7)]
        pairs += [(C + r, C + c) for r in range(7) for c in range(r, 7)]
        return pairs


@pytest.mark.parametrize("C", [32, 64, 128])
def test_index_map_rebuilds_hh_plus_lh_plus_lh_transpose(C):
    lay = Layout(C)
    rng = np.random.default_rng(C)
    X = (rng.standard_normal((96, lay.F)) * np.exp(rng.uniform(-4, 4, lay.F))).astype(np.float32)
    X[:, -1] = 0.0  # the zero feature
    h, l = (a.astype(np.float64) for a in tf32_split(X))
    D = lay.d_of(h, l)
    HH, LH = h.T @ h, l.T @ h
    for i, j in lay.finalize_reads():
        assert D[lay.hh(i, j)] == HH[i, j]
        assert D[lay.lh(i, j)] == LH[i, j] and D[lay.lh(j, i)] == LH[j, i]
    G = emulated_gram(X)
    for i, j in lay.finalize_reads():
        got = (D[lay.hh(i, j)] + D[lay.lh(i, j)]) + D[lay.lh(j, i)]
        assert abs(got - G[i, j]) <= 1e-13 * (np.abs(X[:, i]).astype(np.float64) @ np.abs(X[:, j])), (i, j)


@pytest.mark.parametrize("C", [32, 64, 128])
def test_written_part_of_d_covers_every_finalize_read(C):
    lay = Layout(C)
    written = {n * lay.ROWS + m for m in range(lay.ROWS) for n in range(lay.COLS) if lay.written(m, n)}
    reads = set()
    for i, j in lay.finalize_reads():
        reads |= {lay.hh(i, j), lay.lh(i, j), lay.lh(j, i)}
    assert reads <= written
    # only l*l products are never written, and HH below its diagonal
    for m in range(lay.ROWS):
        for n in range(lay.COLS):
            if not lay.written(m, n):
                (ka, fa), (kb, fb) = lay.a_rows[m], lay.b_cols[n]
                assert (ka, kb) == ("l", "l") or (ka == kb == "h" and fb < fa)
    if C == 32:  # the shipped C = 32 layout: 64 x 56, rows 0-23 of columns 40-55 unused
        assert (lay.ROWS, lay.COLS, lay.S, lay.F) == (64, 56, 24, 40)


@pytest.fixture(scope="module")
def c128_160():
    pair = case_pair(160, 120, 128)
    L = pair.levels[0]
    ref = level_reference(pair, L)
    X, _ = valid_rows(pair, L)
    return ref, X


@pytest.mark.parametrize("cs", [64, 128])
def test_split_tf32_sits_far_below_the_bars(cs):
    pair = case_pair(160, 120, cs)
    L = pair.levels[0]
    ref = level_reference(pair, L)
    X, _ = valid_rows(pair, L)
    e = assert_system_close(gram_result(emulated_gram(X), ref.inliers), ref, ref.S, ref.B, f"split-tf32 C={cs}")
    assert e["h"] <= H_BAR / 50 and e["jtr"] <= JTR_BAR / 50


def test_comparator_rejects_lost_low_rows_of_the_b_side_code_features_at_c128(c128_160):
    """code features 120-127 keep their l rows in B (TcCfg::lh, second branch): losing them is caught"""
    ref, X = c128_160
    _rejected(gram_result(emulated_gram(X, drop_lo=range(12 + 120, 12 + 128)), ref.inliers), ref, "lo 120-127 lost")


def test_comparator_rejects_a_missing_lh_transpose_at_c128(c128_160):
    ref, X = c128_160
    _rejected(gram_result(emulated_gram(X, lh_t=False), ref.inliers), ref, "LH^T missing C=128")
