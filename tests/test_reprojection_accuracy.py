"""Per-entry accuracy of the reprojection factor (ReprojectionFactor::linearize, dfk_sparse.cu) against fp64 truth: the
factor set, the checks, and, on the CPU, proof that the checks reject plausible kernel bugs.

tests/test_gpu_reprojection_accuracy.py runs the device's single-call rows, batched records and error batch over the
factor set of make_factors() and holds them to the checks of evaluate().  Here the same checks run on the fp64 oracle
rows with one kernel bug emulated at a time in numpy: each bug must be rejected by 4x or more, and the weight written
with log1pf (the form the kernel uses) must be accepted.

The checks, for every valid match m of a factor (err = |tr - u| in fp64, s = (err / delta)^2, sigma, w the Cauchy weight
w = a / sqrt(2) sqrt(log1p(1 / a^2)), a = delta / err):

  * Rounding of u.  The device computes u, v in fp32: the warp, the division by Z and fx X / Z + u0 each round at about
    eps times |u - u0| + |u0| + fx |P| / Z, and d = tr - u rounds at eps (|tr| + |u|).  So with
        U_m = |u| + |v| + |tr_x| + |tr_y| + fx + fy
    (fx |P| / Z <= fx (|xn| + |yn| + 1) is at most a few fx in the image; |u0| <= |u| + fx in it), the device's err
    carries an absolute error of at most K_ROUND eps U_m: it cancels in tr - u, so its relative error
    K_ROUND eps U_m / err is what the fp32 arithmetic costs, not a kernel fault.
  * Weight per match.  A match's two rows share the factor w / sigma, so the norm of its 12 + C Jacobian columns on the
    device over the fp64 norm is w_dev / w64 (times 1 + a few eps from the columns themselves).  ln w = ln a - ln 2 / 2
    + ln(log1p(s)) / 2 with s = a^-2 = (err / delta)^2, so
        g = d ln w / d ln err = s / ((1 + s) log1p(s)) - 1,
    which runs from -s / 2 (a >> 1: the weight flattens at 1 / sqrt(2)) to -1 (a << 1: w ~ delta / err).  An error
    delta_err in err moves w by |g| delta_err / err, so
        |w_dev / w64 - 1| <= W_BAR + |g| K_ROUND eps U_m / err  =  W_BAR + rho_m.
  * Rows per column block (pose0, pose1, code, b), each against its own block's largest fp64 entry in the factor:
    |r - r64| <= ROW_BAR max|block64| + rho_m |r64| (the weight's share), and for b additionally
    (w64 / sigma) K_ROUND eps U_m (b = d w / sigma carries d's cancellation).  The code columns are jd_c jc_k w / sigma
    with jd_c = f_c (q_c Z - P_c q_2) / Z^2 * dJ (q = R ray): at a small translation the two products nearly cancel,
    so those columns get K_ROUND eps m_c |jc_k| w / sigma on top, m_c the size of the cancelling terms
    (correspondence64).  At the near-identity pose that is a few 1e-5 of the block.
  * Records against the fp64 Gram of the oracle rows (tests/system_accuracy.py bars):
      JtJ: |H - H64| <= H_BAR S + sum_m 2 rho_m |J_m|^T |J_m|  (the weight term: rho_m scales both rows of m);
      Jtr: |Jtr - Jtr64| <= JTR_BAR B + the gap the fp64 Gram of the single call's rows already has to Jtr64 (b
           carries d's cancellation; the rows are checked above, what the reduction adds is held to JTR_BAR);
      residual: within RES_BAR relative beyond the gap the single call's rows already have (b again);
      inliers: exactly the fp32 oracle's valid matches.
  * Error batch: bit for bit the records' residual, so within the residual bar too.

The rows share one per-match function with the records and the error batch, so the three are checked through one set
of rows.  K_ROUND = 4 leaves the device's own u, v rounding (a few ulp) below the allowance.
"""
from __future__ import annotations

import types

import numpy as np
import pytest

from deepfactors_b200 import se3, synth
from oracle import oracle as orc
from system_accuracy import H_BAR, JTR_BAR, RES_BAR, RowGram, pose_jacobians, system_errors

EPS = 2.0 ** -24
W_BAR = 1e-5
ROW_BAR = 1e-5
K_ROUND = 4.0
REP_HUBER = 0.1  # window_opt.REP_HUBER, the delta the mapper's reprojection links use
CODE_SIZES = [8, 16, 32, 64, 128]


def chunk(cs):
    """matches per chunk of the records kernel (RepCfg<C> in dfk_sparse.cu)"""
    return 64 if cs >= 64 else 128


def match_counts(cs):
    """one match, the chunk edges, two chunks and one, and a long chain of chunk sums"""
    ch = chunk(cs)
    return [1, ch - 1, ch, ch + 1, 2 * ch + 1, 20000]


# regime -> (cauchy_delta, kind, low, high): train = fp64 correspondence + an offset of that kind
REGIMES = {
    "noise": (1.5, "normal", 0.7, None),        # the suite's 0.7 px noise, a = delta / err near 1-6
    "huber": (REP_HUBER, "loguniform", 0.3, 10.0),  # the mapper's delta: a << 1
    "exact": (1.5, "loguniform", 1e-4, 1e-2),   # near-exact matches: a >> 1
    "exact_big_delta": (1e3, "loguniform", 1e-4, 1e-2),
    "noise_big_delta": (1e3, "normal", 0.7, None),  # a large delta, the natural way to switch the robust loss off
}


def poses():
    """the reference test poses and a near-identity pair"""
    near = (se3.identity(), se3.make_pose([2e-3, -1e-3, 1.5e-3], [0.01, -0.006, 0.004], np.float32))
    return [synth.reference_test_poses(), near]


def levels(cs):
    """(level, extra pixels of row padding on the device): a pitched 160x120 and an odd unpitched 97x61"""
    return [(synth.make_level(160, 120, cs, seed=12), 3), (synth.make_level(97, 61, cs, seed=13), 0)]


def correspondence64(pose0, pose1, code, cam, prx_orig, prx_jac, query):
    """the fp64 correspondence (u, v) of every query (pixel (int)q, depth decoded from the code), its validity, and the
    magnitude m [M, 2] of the terms that cancel in the code Jacobian's factor jd = d pix1 / d prx (see Truth)"""
    p10, _, _ = orc.relative_pose(np.asarray(pose1, np.float32).astype(np.float64),
                                  np.asarray(pose0, np.float32).astype(np.float64))
    H_, W_ = prx_orig.shape
    q = np.asarray(query, np.float32)
    xi, yi = q[:, 0].astype(np.int64), q[:, 1].astype(np.int64)  # truncation toward zero, as (int) in C
    inside = (xi >= 0) & (yi >= 0) & (xi < W_) & (yi < H_)
    xc, yc = np.clip(xi, 0, W_ - 1), np.clip(yi, 0, H_ - 1)
    prx = prx_orig[yc, xc].astype(np.float64) + prx_jac[yc, xc].astype(np.float64) @ np.asarray(code, np.float64)
    d = 2.0 / prx - 2.0
    fx, fy, u0, v0 = (float(np.float32(x)) for x in (cam.fx, cam.fy, cam.u0, cam.v0))
    ray = np.stack([(xi - u0) / fx, (yi - v0) / fy, np.ones(xi.shape[0])], 1)
    rp = se3.quat_rotate(p10[:4], ray * d[:, None])
    P = rp + p10[4:7]
    Z = P[:, 2]
    uv = np.stack([fx * P[:, 0] / Z + u0, fy * P[:, 1] / Z + v0], 1)
    # jd_c = f_c (q_c Z - P_c q_2) / Z^2 * dJ, q = R ray, dJ = -2 / prx^2: the two products nearly cancel when the
    # translation is small; each rounds at eps times its size, P_c and Z at eps times S = |R pt|_1 + |t|_1
    A = np.abs(ray) @ np.abs(se3.quat_to_matrix(p10[:4])).T
    S = np.abs(rp).sum(1) + np.abs(p10[4:7]).sum()
    dJ = 2.0 / prx ** 2
    m = np.stack([f * (A[:, c] + 2.0 * S / np.abs(Z) * A[:, 2]) for c, f in ((0, fx), (1, fy))], 1) * (dJ / np.abs(Z))[:, None]
    return uv, inside & (Z > 0), m


def _offsets(rng, n, kind, lo, hi):
    if kind == "normal":
        return rng.normal(0.0, lo, (n, 2))
    mag = np.exp(rng.uniform(np.log(lo), np.log(hi), n))
    ang = rng.uniform(0.0, 2 * np.pi, n)
    return np.stack([mag * np.cos(ang), mag * np.sin(ang)], 1)


def make_factors(cs, regime):
    """one factor per match count of match_counts(cs), images, poses and sigma in {0.5, 2} rotating over them, then a
    factor whose points all fall behind the camera.  Factors of 7 or more matches hold a query left of the image, one
    right of it, one at x.999 (truncated to its pixel, not rounded), one at the last column (W - 0.001) and one at
    x = -0.5 (truncated to column 0).  Returns host dicts: the arguments of ReprojectionLinearize (prx_* host arrays)
    plus 'level' (index into levels(cs)), 'uv64' and 'valid64'."""
    delta, kind, lo, hi = REGIMES[regime]
    rng = np.random.default_rng(1000 * cs + sorted(REGIMES).index(regime))
    lvs = levels(cs)
    out = []
    for k, m in enumerate(match_counts(cs)):
        li = (k + len(regime)) % 2
        L = lvs[li][0]
        pose0, pose1 = poses()[(k // 2 + len(regime)) % 2]
        code = (rng.standard_normal(cs) * 0.3).astype(np.float32)
        W_, H_ = L.prx_orig.shape[1], L.prx_orig.shape[0]
        q = np.stack([rng.uniform(4, W_ - 5, m), rng.uniform(4, H_ - 5, m)], 1).astype(np.float32)
        if m >= 7:
            q[1] = [37.999, 21.999]
            q[2] = [W_ - 0.001, 11.25]
            q[3] = [-4.0, 7.0]
            q[4] = [-0.5, 13.5]
            q[5] = [W_ + 3.0, 9.5]
        uv, valid, mjd = correspondence64(pose0, pose1, code, L.cam, L.prx_orig, L.prx_jac, q)
        t = uv + _offsets(rng, m, kind, lo, hi)
        t[~valid] = q[~valid] + 1.0
        out.append(dict(pose0=pose0, pose1=pose1, code0=code, cam=L.cam, prx_orig=L.prx_orig, prx_jac=L.prx_jac,
                        query_xy=q, train_xy=t.astype(np.float32), cauchy_delta=delta, sigma=(0.5, 2.0)[k % 2],
                        level=li, uv64=uv, valid64=valid, mjd=mjd))
    L = lvs[0][0]
    far = se3.make_pose([0, 0, 0], [0, 0, 30.0], np.float32)
    q = np.array([[10.3, 12.9], [40.0, 30.0], [80.5, 60.5]], dtype=np.float32)
    code = np.zeros(cs, np.float32)
    uv, valid, mjd = correspondence64(se3.identity(), far, code, L.cam, L.prx_orig, L.prx_jac, q)
    out.append(dict(pose0=se3.identity(), pose1=far, code0=code, cam=L.cam, prx_orig=L.prx_orig, prx_jac=L.prx_jac,
                    query_xy=q, train_xy=q + 1.0, cauchy_delta=delta, sigma=1.0, level=0, uv64=uv, valid64=valid,
                    mjd=mjd))
    return out


def _oracle_args(f):
    return (f["pose0"], f["pose1"], f["code0"], f["cam"], f["prx_orig"], f["prx_jac"], f["query_xy"], f["train_xy"],
            f["cauchy_delta"], f["sigma"])


class Truth:
    """fp64 truth of one factor: the oracle rows, per-match err, U, g, rho and w, and the fp32 oracle's valid count"""

    def __init__(self, oracle, f):
        cs = f["code0"].shape[0]
        self.n = 12 + cs
        self.rows, _ = oracle.reprojection_rows(*_oracle_args(f), precision="f64")
        # validity does not depend on the train points: count it where the fp32 weight is well defined
        a = list(_oracle_args(f))
        a[7] = np.asarray(f["query_xy"], np.float32) + 1.0
        a[8] = 1.0
        r32, _ = oracle.reprojection_rows(*a, precision="f32")
        self.inliers = int((np.abs(r32[0::2]).sum(1) > 0).sum())
        tr = np.asarray(f["train_xy"], np.float64)
        uv = f["uv64"]
        self.valid = f["valid64"]
        self.err = np.where(self.valid, np.hypot(tr[:, 0] - uv[:, 0], tr[:, 1] - uv[:, 1]), 1.0)
        cam = f["cam"]
        self.U = np.abs(uv).sum(1) + np.abs(tr).sum(1) + float(cam.fx) + float(cam.fy)
        delta = float(np.float32(f["cauchy_delta"]))
        s = (self.err / delta) ** 2
        self.g = s / ((1.0 + s) * np.log1p(s)) - 1.0
        self.rho = np.where(self.valid, np.abs(self.g) * K_ROUND * EPS * self.U / self.err, 0.0)
        a_ = delta / self.err
        self.w = np.where(self.valid, a_ / np.sqrt(2.0) * np.sqrt(np.log1p(1.0 / a_ ** 2)), 0.0)
        self.sigma = float(np.float32(f["sigma"]))
        # the code columns' own cancellation: K_ROUND eps m_c |jc_k| w / sigma (row 2 m + c, column 12 + k)
        jac = np.asarray(f["prx_jac"], np.float64)
        q = np.asarray(f["query_xy"], np.float32)
        xi = np.clip(q[:, 0].astype(np.int64), 0, jac.shape[1] - 1)
        yi = np.clip(q[:, 1].astype(np.int64), 0, jac.shape[0] - 1)
        k = np.where(self.valid[:, None], f["mjd"] * (self.w / self.sigma)[:, None], 0.0).reshape(-1, 1)
        self.code_allow = K_ROUND * EPS * k * np.repeat(np.abs(jac[yi, xi]), 2, axis=0)


BLOCKS = lambda n: (("pose0", slice(0, 6)), ("pose1", slice(6, 12)), ("code", slice(12, n)), ("b", slice(n, n + 1)))


def evaluate(t: Truth, rows, rec, single_rows=None, err_batch=None):
    """every check of the module docstring on one factor.  rows: the device's rows [2M, 13 + C]; rec: its record
    (JtJ dense [n, n], Jtr = -A^T b, residual, inliers); single_rows: the rows whose fp64 Gram gives the Jtr / residual
    gap (default: rows); err_batch: the error batch's (b^T b, inliers).  Returns {check: (ratio / bar, where)}; the
    factor passes when every ratio is <= 1."""
    n = t.n
    rows = np.asarray(rows, np.float64)
    r64 = t.rows
    single = rows if single_rows is None else np.asarray(single_rows, np.float64)
    out = {}
    v = np.flatnonzero(t.valid)
    if v.size:
        J = lambda r: np.sqrt((r[0::2, :n] ** 2).sum(1) + (r[1::2, :n] ** 2).sum(1))
        with np.errstate(divide="ignore", invalid="ignore"):
            ratio = J(rows)[v] / J(r64)[v]
        dev = np.abs(np.nan_to_num(ratio, nan=np.inf) - 1.0)
        lim = W_BAR + t.rho[v]
        k = int(np.argmax(dev / lim))
        out["weight"] = (float(dev[k] / lim[k]), f"match {v[k]}: w_dev / w64 = {ratio[k]:.9f}, err {t.err[v[k]]:.3e} px, "
                                                 f"w64 {t.w[v[k]]:.6e}, allowance {lim[k]:.2e}")
    rho2 = np.repeat(t.rho, 2)[:, None]
    w2 = np.repeat(t.w, 2)[:, None]
    U2 = np.repeat(t.U, 2)[:, None]
    for name, sl in BLOCKS(n):
        blk64 = r64[:, sl]
        scale = np.abs(blk64).max()
        if scale == 0:
            continue
        allow = rho2 * np.abs(blk64)
        if name == "b":
            allow = allow + w2 / t.sigma * K_ROUND * EPS * U2
        if name == "code":
            allow = allow + t.code_allow
        diff = np.nan_to_num(np.abs(rows[:, sl] - blk64), nan=np.inf)
        r = (diff - allow) / (ROW_BAR * scale)
        i, j = np.unravel_index(int(np.argmax(r)), r.shape)
        out[name] = (float(r[i, j]), f"row {i} col {sl.start + j}: got {rows[i, sl.start + j]:.9e} "
                                     f"ref {blk64[i, j]:.9e}, block scale {scale:.3e}")
    if rec is not None and t.inliers > 0:
        g = RowGram(n).add(r64)
        ref = g.reference(t.inliers)
        a = np.abs(r64[:, :n]) * np.sqrt(2.0 * rho2)
        S_eff = ref.S + (a.T @ a) / H_BAR
        s64 = single[:, :n].T @ single[:, n]
        B_eff = ref.B + np.abs(s64 - ref.Jtr) / JTR_BAR
        res_bar = RES_BAR + abs(float(single[:, n] @ single[:, n]) - ref.residual) / ref.residual
        H, Jtr, res, inl = rec
        got = types.SimpleNamespace(JtJ=H, Jtr=-np.asarray(Jtr, np.float64), residual=float(res), inliers=int(inl))
        e = system_errors(got, ref, S_eff, B_eff)
        out["inliers"] = (0.0 if int(inl) == t.inliers else np.inf, f"{int(inl)} vs fp32 oracle {t.inliers}")
        out["jtj"] = (e["h"] / H_BAR, f"entry {e['h_at']}: got {e['Hg'][e['h_at']]:.9e} ref {ref.H[e['h_at']]:.9e}")
        out["jtr"] = (e["jtr"] / JTR_BAR, f"entry {e['jtr_at']}: got {got.Jtr[e['jtr_at']]:.9e} "
                                          f"ref {ref.Jtr[e['jtr_at']]:.9e}")
        out["residual"] = (e["res"] / res_bar, f"got {float(res):.9e} ref {ref.residual:.9e}")
        if err_batch is not None:
            eb, ei = err_batch
            same = np.float32(eb).tobytes() == np.float32(res).tobytes() and int(ei) == int(inl)
            out["error_batch"] = (0.0 if same else np.inf, f"error batch ({float(eb):.9e}, {int(ei)}) vs record "
                                                           f"({float(res):.9e}, {int(inl)})")
    return out


def report(what, checks):
    """prints every check's ratio and the worst one's place; returns (name, (ratio, where)) of the worst"""
    if not checks:
        print(f"{what}: no valid match")
        return "none", (0.0, "")
    worst = max(checks.items(), key=lambda kv: kv[1][0])
    line = ", ".join(f"{k} {v[0]:.2e}" for k, v in checks.items())
    print(f"{what}: ratio / bar: {line}; worst {worst[0]} at {worst[1][1]}")
    return worst


def gram_record(rows, n, inliers):
    """the record of a row set, in fp64: (JtJ, -A^T b, b^T b, inliers)"""
    rows = np.asarray(rows, np.float64)
    return rows[:, :n].T @ rows[:, :n], -(rows[:, :n].T @ rows[:, n]), float(rows[:, n] @ rows[:, n]), inliers


# ------------------------------------------------------------------------------------------------- CPU: the bars
def _w32(t, f, log1p):
    """the fp32 Cauchy weight of every match from the fp32-rounded err, written with log1pf or as the reference does"""
    with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
        err = np.float32(t.err)
        a = np.float32(f["cauchy_delta"]) / err
        s = np.float32(1.0) / a / a
        lg = np.log1p(s) if log1p else np.log(np.float32(1.0) + s)
        w = np.abs(a) / np.sqrt(np.float32(2.0)) * np.sqrt(lg)
    return np.where(t.valid, w.astype(np.float64), 0.0)


def _reweighted(t, w):
    with np.errstate(divide="ignore", invalid="ignore"):
        k = np.where(t.w > 0, w / t.w, 0.0)
    return t.rows * np.repeat(k, 2)[:, None]


def test_fp64_correspondence_is_the_oracles(oracle):
    """the tests' fp64 correspondence is the oracle's: b64 = (tr - u64) w64 / sigma row by row, u64 within 1e-3 of an
    fp32 rounding of the oracle's u"""
    for cs, regime in ((8, "noise"), (64, "exact"), (32, "huber")):
        for f in make_factors(cs, regime)[:-1]:
            t = Truth(oracle, f)
            d = np.asarray(f["train_xy"], np.float64) - f["uv64"]
            want = (d * (t.w / t.sigma)[:, None]).reshape(-1)
            b = t.rows[:, t.n]
            assert (np.abs(b - want) <= np.repeat(t.w / t.sigma * 1e-3 * EPS * t.U, 2)).all()
            assert t.inliers == int(t.valid.sum())
        assert t.valid[[1, 2, 4]].all() and not t.valid[[3, 5]].any()


def test_the_near_exact_regimes_reach_a_much_greater_than_one(oracle):
    for regime, lo in (("exact", 1e2), ("exact_big_delta", 1e4), ("noise_big_delta", 1e2)):
        f = make_factors(8, regime)[-2]
        a = f["cauchy_delta"] / Truth(oracle, f).err
        assert np.median(a) > lo, (regime, np.median(a))
    f = make_factors(8, "huber")[-2]
    assert np.median(REP_HUBER / Truth(oracle, f).err) < 0.1


@pytest.mark.parametrize("cs", [8, 64])
@pytest.mark.parametrize("regime", sorted(REGIMES))
def test_the_bars_accept_the_log1pf_weight(oracle, cs, regime):
    """oracle rows carrying the fp32 weight written with log1pf (from the fp32-rounded err): every check passes"""
    worst = 0.0
    for i, f in enumerate(make_factors(cs, regime)):
        t = Truth(oracle, f)
        rows = _reweighted(t, _w32(t, f, log1p=True))
        ch = evaluate(t, rows, gram_record(rows, t.n, t.inliers))
        report(f"log1pf weight, C={cs} {regime} factor {i}", ch)
        worst = max([worst] + [v[0] for v in ch.values()])
    assert worst <= 1.0


def _bug_rows(t, f, bug):
    """the rows a kernel with `bug` would give (row bugs); None for reduction bugs"""
    n, r = t.n, t.rows.copy()
    if bug == "reference_float_weight":
        return _reweighted(t, _w32(t, f, log1p=False))
    if bug == "weight_on_b_only":
        k = np.where(t.w > 0, 1.0 / np.where(t.w > 0, t.w, 1.0), 0.0)
        r[:, :n] *= np.repeat(k, 2)[:, None]
        return r
    if bug == "sigma_twice":
        return r / t.sigma
    if bug == "code_from_next_pixel":
        jac = np.asarray(f["prx_jac"], np.float64)
        W_ = jac.shape[1]
        q = np.asarray(f["query_xy"], np.float32)
        xi, yi = q[:, 0].astype(np.int64), q[:, 1].astype(np.int64)
        for m in np.flatnonzero(t.valid):
            jc, jn = jac[yi[m], xi[m]], jac[yi[m], min(xi[m] + 1, W_ - 1)]
            for row in (2 * m, 2 * m + 1):
                r[row, 12:n] = (r[row, 12:n] @ jc) / (jc @ jc) * jn
        return r
    if bug == "pose1_column_transposed":
        P0, P1 = pose_jacobians(f["pose0"], f["pose1"])
        A = r[:, 0:6] @ np.linalg.inv(P0)
        r[:, 6 + 4] = (A @ P1.T)[:, 4]  # column 4 of J_pose1 with P1 indexed [j * 6 + k]
        return r
    return None


ROW_BUGS = ["reference_float_weight", "weight_on_b_only", "sigma_twice", "code_from_next_pixel",
            "pose1_column_transposed"]


@pytest.mark.parametrize("bug", ROW_BUGS + ["chunk_dropped", "last_partial_chunk_dropped"])
@pytest.mark.parametrize("cs", [8, 64])
def test_the_bars_reject_emulated_kernel_bugs(oracle, cs, bug):
    """each bug emulated on the fp64 oracle rows must exceed some bar by 4x or more on some factor of its regime.  The
    reference's float weight is a bug only where 1 + 1 / a^2 rounds: the near-exact regime."""
    regime = "exact" if bug == "reference_float_weight" else ("huber" if bug == "pose1_column_transposed" else "noise")
    fs = make_factors(cs, regime)
    worst = (0.0, "")
    for i, f in enumerate(fs[:-1]):
        t = Truth(oracle, f)
        rows = _bug_rows(t, f, bug)
        if rows is not None:
            rec = gram_record(rows, t.n, t.inliers)
        else:
            M = t.valid.shape[0]
            ch = chunk(cs)
            if M != 2 * ch + 1:
                continue
            keep = np.ones(M, bool)
            keep[ch:2 * ch] = bug != "chunk_dropped"
            keep[2 * ch:] = bug == "chunk_dropped"
            rows = t.rows
            rec = gram_record(t.rows[np.repeat(keep, 2)], t.n, t.inliers)
        ch = evaluate(t, rows, rec)
        w = report(f"{bug}, C={cs} {regime} factor {i}", ch)
        if w[1][0] > worst[0]:
            worst = (w[1][0], w[0])
    print(f"{bug}, C={cs}: rejected by {worst[0]:.2e} x its bar on {worst[1]}")
    assert worst[0] >= 4.0, worst
