"""BASELINE.json configs[1] at FULL size (1k cameras / 200k points / 2M observations) through size-independent
properties (the oracle only evaluates the cost here; a full CPU solve at this size is the bench's cpu_baseline job):
initial cost identical to the oracle, monotone decrease over successful steps, convergence to the noise floor
0.5 * sigma^2 * (2 N_obs - dof), symmetry / positive-definiteness / linearity of the reduced operator, and solving twice
gives the same trajectory up to the non-associativity of the fp64 RED accumulations (the CPU oracle on this exact
configuration: 10 LM iterations, final cost 1.0018 x the noise floor, in 17 s on 8 threads).
Written after the round-1 GPU budget was exhausted: first executed by the round-end driver."""
import os

import numpy as np
import pytest

from helpers import rel_err
from theiasfm_b200 import _abi, engine, synthetic

pytestmark = pytest.mark.gpu
KW = dict(use_inner_iterations=0, linear_solver_type=_abi.ITERATIVE_SCHUR, max_num_iterations=30)


def test_config2_full_size_properties(oracle):
    p = synthetic.make_config("c2_1kcam")
    assert p.n_obs == 2_000_000 and p.n_cam == 1000 and p.n_pt == 200_000
    o = oracle.Oracle(p.copy(), oracle.default_options(**KW))
    ok, cost_o = o.linearize()
    o.close()
    eng = engine.Engine()
    eng.upload(p, engine.default_options(**KW))
    ok_g, cost_g = eng.linearize()
    assert ok and ok_g and abs(cost_g - cost_o) <= 1e-11 * cost_o
    assert eng.prepare_linear_system(1e4)
    rng = np.random.default_rng(0)
    free_i = np.zeros(10); free_i[[0, 5, 6]] = 1
    a = (rng.normal(size=p.n_cam * 6), rng.normal(size=10) * free_i)
    b = (rng.normal(size=p.n_cam * 6), rng.normal(size=10) * free_i)
    Sa, Sb = eng.schur_matvec(*a), eng.schur_matvec(*b)
    dot = lambda u, v: float(u[0] @ v[0] + u[1] @ v[1])
    assert abs(dot(a, Sb) - dot(b, Sa)) <= 1e-9 * abs(dot(a, Sb)) and dot(a, Sa) > 0
    Sab = eng.schur_matvec(a[0] - 2 * b[0], a[1] - 2 * b[1])
    assert rel_err(Sab[0], Sa[0] - 2 * Sb[0]) < 1e-10
    s1 = eng.minimize()
    assert s1.success
    costs = [i["cost"] for i in s1.iterations if i["step_is_successful"]]
    assert all(y <= x for x, y in zip(costs, costs[1:]))
    dof = 6 * p.n_cam + 3 + 3 * p.n_pt  # gauge-free degrees of freedom, roughly
    floor = 0.5 * 0.25 * (2 * p.n_obs - dof)
    assert 0.9 * floor < s1.final_cost < 1.25 * floor, (s1.final_cost, floor, s1.message)
    # same problem again from the same start: identical control flow, costs equal to RED-order rounding
    q = synthetic.make_config("c2_1kcam")
    s2 = eng.solve(q, engine.default_options(**KW))
    eng.close()
    assert abs(s2.num_iterations - s1.num_iterations) <= 1
    n = min(len(s1.costs), len(s2.costs))
    assert np.all(np.abs(s2.costs[:n] - s1.costs[:n]) <= 1e-7 * s1.costs[:n])


@pytest.mark.parametrize("workload,n_obs,iters", [("c2_1kcam", 2_000_000, 6), ("c4_radtan", 5_000_000, 5)])
def test_full_size_trajectory_matches_oracle(oracle, workload, n_obs, iters):
    """BASELINE.json configs[1] and configs[3] at FULL size: the first LM iterations against the CPU oracle -- per-iteration cost,
    PCG iteration counts, step acceptance and the parameters after the last iteration.  configs[3] is the only full-size run of
    the per-camera-intrinsics-group code path (1000 groups of PINHOLE_RADIAL_TANGENTIAL, pinhole_radial_tangential_camera_model.h:190-291):
    non-shared intrinsics columns in the matvec / rhs / SCHUR_JACOBI blocks.  Tolerances: 1e-9 relative on the costs (fp64
    summation order only; the PCG takes the same number of iterations), 1e-6 on the parameters."""
    kw = dict(use_inner_iterations=0, linear_solver_type=_abi.ITERATIVE_SCHUR, max_num_iterations=iters)
    p0 = synthetic.make_config(workload)
    assert abs(p0.n_obs - n_obs) <= 0.01 * n_obs
    oracle.set_num_threads(min(32, len(os.sched_getaffinity(0))))
    po, pg = p0.copy(), p0.copy()
    so = oracle.solve(po, oracle.default_options(**kw))
    eng = engine.Engine()
    sg = eng.solve(pg, engine.default_options(**kw))
    eng.close()
    assert sg.rc == 0 and sg.success and so.success
    assert abs(sg.initial_cost - so.initial_cost) <= 1e-11 * so.initial_cost
    assert sg.num_iterations == so.num_iterations == iters + 1
    assert [i["linear_solver_iterations"] for i in sg.iterations] == [i["linear_solver_iterations"] for i in so.iterations]
    assert [i["step_is_successful"] for i in sg.iterations] == [i["step_is_successful"] for i in so.iterations]
    ok = np.array([bool(i["step_is_successful"]) for i in so.iterations])
    rel = np.abs(sg.costs - so.costs) / so.costs
    # accepted steps: 1e-9.  A REJECTED step's cost is the cost of an overshooting candidate far outside the region where the
    # quadratic model holds: the rounding-level difference of the two inexact PCG solutions is amplified there (2.3e-8 measured on
    # the GPU for iteration 3 of config 2, between neighbours that agree to 7e-13 and 7e-10) -- 1e-6 for those
    assert np.all(rel[ok] <= 1e-9) and np.all(rel <= 1e-6), (sg.costs, so.costs)
    assert rel_err(pg.ext, po.ext) < 1e-6 and rel_err(pg.pt, po.pt) < 1e-6 and rel_err(pg.intr, po.intr) < 1e-6
