"""States and observations that make Evaluator::Evaluate fail -- or, just as deliberately, not fail -- shared by the GPU
tests (tests/test_gpu_eval_failure.py) and by their CPU guard on the oracle alone (tests/test_oracle_eval_failure_cases.py),
which fails if a change here stops a construction from doing what it is built for.

The reference's rules (residual_block.cc:100-131, program_evaluator.h:205-292; the oracle restates them in
oracle/bal.h:336-423): residuals are always checked; the Jacobian is checked whenever it is computed, i.e. when the
Jacobian or the gradient is asked for; the summed cost must be finite; all of it before the loss's Corrector.

Every bad value is built so that GPU and oracle compute it the same way, with a margin of orders of magnitude, so that
no verdict depends on summation order, sincos against sin / cos or norm3d against hypot.  The three main kinds sit on a
camera whose angle-axis and translation are exactly zero: rotation takes the first-order branch (rotation.h:874,
kernels.cuh snavely), p = X + w x X + t = X exactly on both sides, and the target row's point X is then placed directly
in the camera frame:

  residual_nonfinite  X_z = 0: x_p = -X_x / 0, a non-finite residual in every call mode.
  jacobian_only       X = (-1e-307, 0, 1e-307), f = 800, l1 = l2 = 0: x_p is 1 to the last bit or two, the residual is
                      finite, but d r / d X_z contains f / p_z = 8e309 = inf.  Every mode that computes J fails, cost-only
                      and residual-only calls succeed.
  cost_overflow       X = (-1.2e151, 0, 1), f = 1e3, l1 = l2 = 0 on k rows: r_x = 1.2e154 - o_x, each row costs
                      0.72e308.  Two rows sum below 0.9 DBL_MAX and succeed; three overflow, but only in the final sum
                      (no row, and no partial sum of two, reaches DBL_MAX), so cost-only and residual-only calls fail on
                      the host's isfinite(cost) alone.  Under Huber(a) the cost grows linearly (rho = 2 a |r| - a^2), so
                      three rows succeed.  d r / d l1 = f r2 x_p = inf: every mode that computes J fails anyway.

The plain kinds put NaN or +-inf into one point coordinate or one camera intrinsic (every row of that camera fails), and
with_observation() into one observation, which is given at b200_create.  These fail in every mode.

The LM loop's own failure path (a candidate whose evaluation fails counts as an unsuccessful step,
trust_region_minimizer.cc) is not built here: only the pole at p_z = 0 makes a candidate non-finite, and a candidate
within ~1e-300 of it cannot be placed so that two summation orders of the step agree on which side of it it lands.
"""
import numpy as np

DBL_MAX = np.finfo(np.float64).max

# name -> (want_residuals, want_gradient, want_jacobian), the arguments of Problem.evaluate / BaProgram.evaluate
MODES = {
    "cost": (False, False, False),
    "residuals": (True, False, False),
    "gradient": (True, True, False),
    "gradient_jacobian": (True, True, True),
    "jacobian": (False, False, True),
}
J_MODES = ("gradient", "gradient_jacobian", "jacobian")   # the modes that compute J

PLAIN_KINDS = ("point_nan", "point_inf", "camera_nan", "camera_inf")
OBSERVATION_KINDS = ("observation_nan", "observation_inf")

OVERFLOW_X = (-1.2e151, 0.0, 1.0)
OVERFLOW_INTRINSICS = (1e3, 0.0, 0.0)
JACOBIAN_ONLY_X = (-1e-307, 0.0, 1e-307)
JACOBIAN_ONLY_INTRINSICS = (800.0, 0.0, 0.0)


def expected_ok(kind, mode, huber=False):
    """The verdict of Evaluate for a construction of `kind` called in `mode`, under Huber or the trivial loss."""
    if kind in ("jacobian_only", "cost_overflow2"):
        return mode not in J_MODES
    if kind == "cost_overflow3":
        return mode not in J_MODES and huber
    return False


def overflow_count(kind):
    return {"cost_overflow2": 2, "cost_overflow3": 3}.get(kind, 1)


def affected_rows(row_cam, row_pt, rows):
    """Rows whose camera is one of the target rows' cameras and whose point is one of their points: each of them sees
    its point directly in the frame of a zeroed camera."""
    cams = np.unique(np.asarray(row_cam)[rows])
    pts = np.unique(np.asarray(row_pt)[rows])
    return np.flatnonzero(np.isin(row_cam, cams) & np.isin(row_pt, pts))


def overflow_rows(row_cam, row_pt, candidates, k):
    """k of `candidates` (rows, in order of preference) with distinct points and no duplicate (camera, point) pair, such
    that exactly these k rows see a target point through a zeroed camera."""
    out = []
    for r in candidates:
        trial = out + [int(r)]
        if len(affected_rows(row_cam, row_pt, trial)) == len(trial):
            out = trial
            if len(out) == k:
                return out
    raise AssertionError("no %d independent rows among %s" % (k, list(candidates)))


def construct(state, row_cam, row_pt, P, kind, rows):
    """`state` (points [3P], then cameras [9C]) with the bad value of `kind` at the target rows `rows`: one row for every
    kind but cost_overflow2 / cost_overflow3, which take 2 and 3 rows from overflow_rows()."""
    x = np.array(state, dtype=float, copy=True)
    rows = [int(r) for r in np.atleast_1d(rows)]
    assert len(rows) == overflow_count(kind), (kind, rows)
    cam_ofs = [3 * P + 9 * int(row_cam[r]) for r in rows]
    pt_ofs = [3 * int(row_pt[r]) for r in rows]
    if kind == "point_nan":
        x[pt_ofs[0]] = np.nan
    elif kind == "point_inf":
        x[pt_ofs[0] + 2] = np.inf
    elif kind == "camera_nan":
        x[cam_ofs[0] + 6] = np.nan       # f
    elif kind == "camera_inf":
        x[cam_ofs[0] + 7] = -np.inf      # l1
    else:
        for c in cam_ofs:
            x[c:c + 6] = 0.0
        for c, p in zip(cam_ofs, pt_ofs):
            if kind == "residual_nonfinite":
                x[p + 2] = 0.0
            elif kind == "jacobian_only":
                x[c + 6:c + 9] = JACOBIAN_ONLY_INTRINSICS
                x[p:p + 3] = JACOBIAN_ONLY_X
            else:
                x[c + 6:c + 9] = OVERFLOW_INTRINSICS
                x[p:p + 3] = OVERFLOW_X
        if kind.startswith("cost_overflow"):
            assert len(affected_rows(row_cam, row_pt, rows)) == len(rows), rows
    return x


def zeroed_cameras(state, row_cam, P, kind, rows):
    """The healthy part of a construction: its cameras zeroed (and their intrinsics set), its points left as they are.
    Every row of it must evaluate, which the CPU guard asserts."""
    x = np.array(state, dtype=float, copy=True)
    intrinsics = {"jacobian_only": JACOBIAN_ONLY_INTRINSICS}.get(kind, OVERFLOW_INTRINSICS)
    for r in np.atleast_1d(rows):
        c = 3 * P + 9 * int(row_cam[r])
        x[c:c + 6] = 0.0
        if kind != "residual_nonfinite":
            x[c + 6:c + 9] = intrinsics
    return x


def overflow_row_cost(obs_xy):
    """0.5 |r|^2 of a cost_overflow row with observation obs_xy: r = (f x_p - o_x, -o_y) with x_p = 1.2e151."""
    rx = OVERFLOW_INTRINSICS[0] * -OVERFLOW_X[0] - obs_xy[0]
    return 0.5 * (rx * rx + obs_xy[1] * obs_xy[1])


def with_observation(bal, obs_of_row, row, kind):
    """`bal` with o_x of reduced-program row `row` NaN (observation_nan) or its o_y -inf (observation_inf): both the GPU
    library and the oracle take the observations at construction."""
    from ceres_solver_b200 import bal as B
    obs = np.array(bal.obs, dtype=float, copy=True)
    i = int(obs_of_row[row])
    if kind == "observation_nan":
        obs[i, 0] = np.nan
    else:
        obs[i, 1] = -np.inf
    return B.Bal(bal.cam_idx, bal.pt_idx, obs, bal.cameras, bal.points)


def zeroable_cameras(state, row_cam, row_pt, P):
    """Cameras that can be zeroed: once p = X, every point they see is clear of the camera plane, |X_z| > 1e-3 (1 + |X_x|
    + |X_y|).  A normalized BAL problem has points with X_z exactly 0 (the median is subtracted)."""
    X = np.asarray(state[:3 * P]).reshape(P, 3)[np.asarray(row_pt)]
    clear = np.abs(X[:, 2]) > 1e-3 * (1.0 + np.abs(X[:, 0]) + np.abs(X[:, 1]))
    C = int(np.max(row_cam)) + 1
    return np.bincount(row_cam, weights=~clear, minlength=C) == 0


def placements(state, row_cam, row_pt, P, perm, seed=0, ordinary=3, big=2):
    """{label: row} of the target rows of a problem: a row of the first and of the last point of the internal order
    `perm` (b200_plan_point_order: perm[k] is the point at internal position k), of up to `big` points of 33..128 and of
    more than 128 rows (the chunk tiles), of a degree-1 point, a duplicated (camera, point) row, and of a seeded sample of
    ordinary points.  Each is the first row of its point whose camera is zeroable (the duplicate: the second row of the
    pair); "first" and "last" move inwards along `perm` until there is one."""
    row_cam = np.asarray(row_cam)
    row_pt = np.asarray(row_pt)
    deg = np.bincount(row_pt, minlength=P)
    ptr = np.concatenate([[0], np.cumsum(deg)])
    usable = zeroable_cameras(state, row_cam, row_pt, P)[row_cam]
    first_usable = np.full(P, -1, dtype=np.int64)
    for r in np.flatnonzero(usable)[::-1]:
        first_usable[row_pt[r]] = r
    has = first_usable >= 0
    rng = np.random.RandomState(seed)
    out = {"first": int(first_usable[next(j for j in perm if has[j])]),
           "last": int(first_usable[next(j for j in perm[::-1] if has[j])])}
    for name, lo, hi in (("rows33_128", 33, 128), ("rows129+", 129, 1 << 30)):
        pts = np.flatnonzero((deg >= lo) & (deg <= hi) & has)
        for i, j in enumerate(sorted(rng.choice(pts, size=min(big, pts.size), replace=False))):
            out["%s_%d" % (name, i)] = int(first_usable[j])
    ones = np.flatnonzero((deg == 1) & has)
    if ones.size:
        out["degree1"] = int(first_usable[ones[0]])
    key = row_pt.astype(np.int64) * (int(row_cam.max()) + 1) + row_cam
    _, first, counts = np.unique(key, return_index=True, return_counts=True)
    dups = [k for k in first[counts > 1] if usable[k]]
    if dups:
        out["duplicate"] = int(np.flatnonzero(key == key[dups[0]])[-1])   # the second row of the pair
    plain = np.flatnonzero((deg >= 2) & (deg <= 32) & has)
    for i, j in enumerate(sorted(rng.choice(plain, size=min(ordinary, plain.size), replace=False))):
        out["ordinary_%d" % i] = int(first_usable[j])
    return out


def overflow_candidates(places, state, row_cam, row_pt, P, seed=0):
    """Candidate target rows for cost_overflow, far apart in row order: the placement rows sorted, then taken
    alternately from both ends inwards; then every row with a zeroable camera in a seeded order (on a problem with few
    cameras, most pairs of points are seen by each other's cameras)."""
    rows = sorted(set(places.values()))
    order = []
    while rows:
        order.append(rows.pop(0))
        if rows:
            order.append(rows.pop())
    usable = zeroable_cameras(state, row_cam, row_pt, P)[np.asarray(row_cam)]
    return order + [int(r) for r in np.random.RandomState(seed).permutation(np.flatnonzero(usable))]


def overflow_targets(places, state, row_cam, row_pt, P):
    """The three cost_overflow rows of a problem (cost_overflow2 takes the first two)."""
    return overflow_rows(row_cam, row_pt, overflow_candidates(places, state, row_cam, row_pt, P), 3)
