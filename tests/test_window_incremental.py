"""CPU tests of IncrementalOptimizer (the ISAM2 update rule: relinearisation threshold and skip, theta_lin bookkeeping,
the returned counts) on a fake problem, of the growth rule of dfk_window_solver_create_from (reusable_columns), and of
IncrementalOptimizer driving OptimizeWork through signal_no_relinearize."""
import numpy as np
import pytest

from deepfactors_b200 import se3
from deepfactors_b200.factors import WindowBlocks
from deepfactors_b200.window_opt import (IncrementalOptimizer, OptimizeWork, level_at, level_start, reusable_columns,
                                         solver_columns)

CS = 4
B = 6 + CS


def lastn_pairs(K, n):
    return [p for k in range(1, K) for m in range(max(0, k - n), k) for p in ((k, m), (m, k))]


class Fake:
    """linearise returns a diagonal buffer and records what it was asked; solve returns scripted deltas"""

    def __init__(self, layout, deltas, first_columns=None):
        self.layout, self.deltas = layout, list(deltas)
        self.first_columns = list(first_columns or [0] * len(self.deltas))
        self.calls = []

    def linearise(self, poses, codes, todo, frame_poses=None):
        self.calls.append((poses.copy(), codes.copy(), None if frame_poses is None else frame_poses.copy(), list(todo)))
        buf = np.zeros(self.layout.floats, np.float32)
        K = self.layout.num_keyframes
        D = buf[:K * B * B].reshape(K, B, B)
        D[:] = np.eye(B, dtype=np.float32) * 2.0
        D[1, 3, 3] = 4.0e6
        return buf, None

    def solve(self, buf, diag_eps, codes):
        self.eps = diag_eps
        return self.deltas.pop(0), self.first_columns.pop(0)


def setup(K=3, F=0, deltas=(), first_columns=None, **kw):
    pairs = [(k, k + 1) for k in range(K - 1)] + [(0, K + f) for f in range(F)]
    layout = WindowBlocks(K, CS, pairs, num_frames=F)
    fake = Fake(layout, deltas, first_columns)
    poses = np.tile([0, 0, 0, 1.0, 0.1, 0.2, 0.3], (K, 1))
    codes = np.zeros((K, CS))
    frames = np.tile([0, 0, 0, 1.0, 0, 0, 1.0], (F, 1)) if F else None
    opt = IncrementalOptimizer(layout, fake.linearise, fake.solve, poses, codes, frames, **kw)
    return opt, fake, layout


def delta(layout, entries):
    d = np.zeros(layout.dim)
    for i, v in entries.items():
        d[i] = v
    return d


def test_threshold_is_inclusive_and_pose_and_code_are_separate_keys():
    K = 3
    layout = WindowBlocks(K, CS, [(0, 1), (1, 2)])
    d1 = delta(layout, {B + 2: 0.05,            # keyframe 1's pose at exactly the threshold: relinearised
                        B + 7: 0.0499999,       # keyframe 1's code just below: not
                        2 * B + 6 + 3: -0.06,   # keyframe 2's code (negative): relinearised
                        2 * B + 1: 0.01})       # keyframe 2's pose: not
    opt, fake, _ = setup(K, deltas=[d1, np.zeros(layout.dim)])
    r = opt.update()
    assert r.variables_relinearized == 0  # the first update has no delta yet
    assert opt.relinearize_keys() == [("pose", 1), ("code", 2)]
    p0, c0 = opt.lin_poses.copy(), opt.lin_codes.copy()
    r = opt.update()
    assert r.variables_relinearized == 2
    assert np.array_equal(opt.lin_poses[1], se3.retract(p0[1], d1[B:B + 6], np.float64))
    assert np.array_equal(opt.lin_poses[[0, 2]], p0[[0, 2]])  # bit for bit: keyframe 2's pose stays
    assert np.array_equal(opt.lin_codes[2], c0[2] + d1[2 * B + 6:3 * B])
    assert np.array_equal(opt.lin_codes[:2], c0[:2])
    # the second linearisation is at theta_lin, and re-evaluates exactly the factors on a relinearised key
    # (pair (0, 1): pose1 moved; pair (1, 2): pose0 moved; keyframe 2's code is code1 of no pair)
    assert np.array_equal(fake.calls[1][0], opt.lin_poses)
    assert fake.calls[0][3] == [0, 1] and fake.calls[1][3] == [0, 1]


def test_counts_and_estimate():
    K = 3
    layout = WindowBlocks(K, CS, [(0, 1), (1, 2)])
    d1 = delta(layout, {2 * B + 6: 0.2})
    d2 = delta(layout, {B + 6: 0.001})
    opt, fake, _ = setup(K, deltas=[d1, d2, d2], first_columns=[0, 2, 3])
    r = opt.update()
    assert (r.variables_relinearized, r.variables_reeliminated, r.factors_relinearised, r.first_column) == \
        (0, 3 * B, 2, 0)
    est = opt.estimate()
    assert np.allclose(est[1][2], d1[2 * B + 6:3 * B])
    r = opt.update()  # keyframe 2's code relinearised; it is code1 of pair (1, 2) only: no factor depends on it
    assert (r.variables_relinearized, r.variables_reeliminated, r.factors_relinearised, r.first_column) == \
        (1, B, 0, 2)
    assert np.array_equal(opt.lin_codes[2], d1[2 * B + 6:3 * B])
    r = opt.update()
    assert (r.variables_relinearized, r.variables_reeliminated, r.factors_relinearised) == (0, 0, 0)
    # estimate = theta_lin (+) delta
    p, c, _ = opt.estimate()
    assert np.array_equal(c[1], opt.lin_codes[1] + d2[B + 6:2 * B])
    # diag_eps: 1e-12 max|d| of the first linearisation over the kept variables, fixed afterwards
    assert fake.eps == 1e-12 * 4.0e6


def test_relinearize_skip():
    K = 2
    layout = WindowBlocks(K, CS, [(0, 1)])
    big = delta(layout, {B: 0.5})
    opt, fake, _ = setup(K, deltas=[big] * 6, relinearize_skip=3)
    moved = [opt.update().variables_relinearized for _ in range(6)]
    assert moved == [0, 0, 1, 0, 0, 1]  # updates 3 and 6 check (GTSAM: ++count % skip == 0)
    with pytest.raises(ValueError):
        setup(K, relinearize_skip=0)


def test_frames_are_keys_of_their_own():
    K, F = 2, 2
    opt, fake, layout = setup(K, F, deltas=[None, None])
    fake.deltas = [delta(layout, {K * B + 6 + 2: 0.3}), np.zeros(layout.dim)]
    opt.update()
    assert opt.relinearize_keys() == [("frame", 1)]
    f0 = opt.lin_frames.copy()
    r = opt.update()
    assert r.variables_relinearized == 1 and r.factors_relinearised == 1  # the frame's pair only
    assert fake.calls[1][3] == [2]  # pairs: (0, 1), then the frames' (0, K), (0, K + 1)
    assert np.array_equal(opt.lin_frames[1], se3.retract(f0[1], np.r_[0, 0, 0.3, 0, 0, 0], np.float64))
    assert np.array_equal(opt.lin_frames[0], f0[0])
    assert r.variables_reeliminated == K * B + 6 * F


def test_grow_keeps_the_cache_and_the_points():
    K = 3
    opt, fake, layout = setup(K, deltas=[delta(WindowBlocks(K, CS, []), {6: 0.01})])
    opt.update()
    new = WindowBlocks(K + 1, CS, layout.pairs + [(3, 2), (2, 3)])
    fake2 = Fake(new, [np.zeros(new.dim)])
    poses = np.tile([0, 0, 0, 1.0, 9, 9, 9], (K + 1, 1))
    codes = np.full((K + 1, CS), 0.5)
    lp = opt.lin_poses.copy()
    opt.grow(new, fake2.linearise, poses, codes, solve=fake2.solve)
    assert np.array_equal(opt.lin_poses[:K], lp) and np.array_equal(opt.lin_poses[K], poses[K])
    assert np.array_equal(opt.lin_codes[K], codes[K])
    assert opt.delta[6] == 0.01 and opt.delta.size == new.dim
    r = opt.update()
    assert fake2.calls[0][3] == [2, 3] and r.factors_relinearised == 2  # the new factors only
    with pytest.raises(ValueError):
        opt.grow(WindowBlocks(K, CS, layout.pairs), fake2.linearise, poses, codes, solve=fake2.solve)


# ------------------------------------------------------------------------------------------------ growth rule
def test_solver_columns_match_the_symbolic_fill():
    cols = solver_columns(5, [(0, 2), (4, 0), (1, 2)], [(3, 1)])
    assert cols == [[2, 4], [2, 3], [3, 4], [4], []]


@pytest.mark.parametrize("n", [1, 4])
def test_appended_keyframe_reuses_all_but_its_back_connections(n):
    for K in (6, 10):
        old = WindowBlocks(K, CS, lastn_pairs(K, n))
        new = WindowBlocks(K + 1, CS, lastn_pairs(K + 1, n))
        assert reusable_columns(old, new) == max(K - n, 0)
        # pairs added in any order, one direction only: the same columns
        one_way = WindowBlocks(K + 1, CS, old.pairs + [(K, K - m) for m in range(1, n + 1)])
        assert reusable_columns(old, one_way) == K - n


def test_full_connections():
    K = 6
    full = [(a, b) for a in range(K) for b in range(K) if a != b]
    old = WindowBlocks(K, CS, full)
    new = WindowBlocks(K + 1, CS, full + [(K, m) for m in range(K)])
    assert reusable_columns(old, new) == 0
    # FULL connections after a keyframe joined to the last one only: column K - 1 is the first changed
    new1 = WindowBlocks(K + 1, CS, full + [(K, K - 1)])
    assert reusable_columns(old, new1) == K - 1


def test_loop_link_between_old_keyframes():
    K = 10
    old = WindowBlocks(K, CS, lastn_pairs(K, 4))
    assert reusable_columns(old, WindowBlocks(K, CS, old.pairs, [(K - 1, 2)])) == 2
    assert reusable_columns(old, WindowBlocks(K, CS, old.pairs + [(2, K - 1)])) == 2
    # a link inside the existing band changes nothing
    assert reusable_columns(old, WindowBlocks(K, CS, old.pairs, [(5, 3)])) == K
    # grown and closed at once: the smaller of the two
    assert reusable_columns(old, WindowBlocks(K + 1, CS, lastn_pairs(K + 1, 4), [(K, 1)])) == 1


def test_tracked_frames_and_priors():
    K = 8
    old = WindowBlocks(K, CS, lastn_pairs(K, 2) + [(3, K)], num_frames=1)
    # a frame added or marginalised makes no tile: every column is reusable (its data change shows at the update)
    assert reusable_columns(old, WindowBlocks(K, CS, lastn_pairs(K, 2) + [(3, K), (5, K + 1)], num_frames=2)) == K
    assert reusable_columns(old, WindowBlocks(K, CS, lastn_pairs(K, 2))) == K
    # a keyframe prior over (1, 4, 6) joins column 1 to 4 and 6
    assert reusable_columns(old, WindowBlocks(K, CS, lastn_pairs(K, 2), kf_priors=[(1, 4, 6)])) == 1


def test_rejects_windows_that_do_not_extend():
    K = 6
    old = WindowBlocks(K, CS, lastn_pairs(K, 2))
    fixed = list(range(6))
    with pytest.raises(ValueError):
        reusable_columns(old, WindowBlocks(K - 1, CS, lastn_pairs(K - 1, 2)), fixed, fixed)
    with pytest.raises(ValueError):
        reusable_columns(old, WindowBlocks(K + 1, 8, lastn_pairs(K + 1, 2)), fixed, fixed)
    with pytest.raises(ValueError):
        reusable_columns(old, WindowBlocks(K + 1, CS, lastn_pairs(K + 1, 2)), fixed, [])
    with pytest.raises(ValueError):
        reusable_columns(old, WindowBlocks(K + 1, CS, lastn_pairs(K + 1, 2)), fixed, fixed + [B])
    # fixing a new keyframe's variable is fine
    assert reusable_columns(old, WindowBlocks(K + 1, CS, lastn_pairs(K + 1, 2)), fixed, fixed + [K * B]) == K - 2


# ------------------------------------------------------------------------------------ driving OptimizeWork
@pytest.mark.parametrize("iters", [[4, 8, 15], [2, 0, 3]])
def test_incremental_optimizer_drives_optimize_work(iters):
    """Mapper::MappingStep's loop: bookkeeping, ISAM2 update, work update, then signal_no_relinearize when the update
    relinearised nothing.  The level each step's factor holds follows the transliteration's rule (level_at with a stall
    jumping to the next finer level's start)."""
    K = 2
    layout = WindowBlocks(K, CS, [(0, 1)])
    rng = np.random.default_rng(sum(iters))
    total = sum(i + 1 for i in iters) + 4
    # scripted deltas: some steps move keyframe 1's pose past the threshold, the others not
    big = [bool(rng.uniform() < 0.5) for _ in range(total)]
    deltas = [delta(layout, {B: 0.1 if b else 0.001}) for b in big]
    opt, fake, _ = setup(K, deltas=deltas)
    w, s = OptimizeWork(iters), 0
    seen = []
    for step in range(total):
        f = w.bookkeeping()
        assert (-1 if f is None else f) == level_at(iters, s), step
        seen.append(f)
        r = opt.update()
        w.update()
        s += 1 if level_at(iters, s) >= 0 else 0
        # the update relinearised exactly when the previous delta was large
        assert r.variables_relinearized == (1 if step > 0 and big[step - 1] else 0), step
        if r.variables_relinearized == 0:
            w.signal_no_relinearize()
            lvl = level_at(iters, s)
            if lvl <= 0:  # a stall at the finest level ends the work
                assert w.finished()
                break
            s = level_start(iters, lvl - 1)
    assert seen[0] == len(iters) - 1 and len(seen) > 1
