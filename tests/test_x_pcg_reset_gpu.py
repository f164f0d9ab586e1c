"""The residual reset of ITERATIVE_SCHUR's conjugate gradients against the oracle.

Every cg_residual_reset_period iterations the CG loop replaces the recurrence r -= alpha q by the true residual r = b - S x, one
extra matvec (ConjugateGradientsSolver; ba_oracle.c).  On the GPU that is its own sequence of vector phases around the extra
matvec: xs = sm .* x and y = 0 before it; the fold (or peer-memory sum) of its y, the fresh residual, z = M^-1 r and the partial
sums behind it.  Periods 1, 3 and 10 reset on every iteration, between iterations and once or twice per solve; eta is small
enough that one of the two solves of each scene runs at least ten iterations.  Three scenes: one shared intrinsics group (the replica rows of the matvec
are folded inside the vector phases), per-camera groups, and the IDENTITY preconditioner.  Each walks the linear system at two
trust-region radii block by block (helpers.block_err), with the tolerances of test_x_long_tracks_gpu."""
import numpy as np
import pytest

from helpers import block_err
from theiasfm_b200 import _abi, engine, synthetic

pytestmark = pytest.mark.gpu

SCENES = {
    "pinhole_shared": dict(scene=dict(n_cam=12, n_pt=300, obs_per_pt=6, seed=71)),
    "radtan_per_camera": dict(scene=dict(n_cam=12, n_pt=300, obs_per_pt=6, model=_abi.MODEL_PINHOLE_RADIAL_TANGENTIAL,
                                         shared_intrinsics=False, seed=72)),
    # without a preconditioner CG needs about twice the iterations for the same eta, and its step drifts from the oracle's at 1e-4
    "identity_precond": dict(scene=dict(n_cam=12, n_pt=300, obs_per_pt=6, seed=73),
                             options=dict(preconditioner_type=_abi.PRECOND_IDENTITY), eta=3e-3),
}
STEPS = ((_abi.VEC_STEP_CAM, 6), (_abi.VEC_STEP_INTR, 10), (_abi.VEC_STEP_PT, 4))


def _opts(mod, name, **kw):
    o = dict(use_inner_iterations=0, linear_solver_type=_abi.ITERATIVE_SCHUR)
    o.update(SCENES[name].get("options", {}))
    o.update(kw)
    return mod.default_options(**o)


@pytest.fixture(scope="module")
def eng():
    e = engine.Engine()
    yield e
    e.close()


@pytest.mark.parametrize("period", [1, 3, 10])
@pytest.mark.parametrize("name", list(SCENES))
def test_residual_reset_stage_parity(eng, oracle, name, period):
    p = synthetic.make_scene(**SCENES[name]["scene"])
    kw = dict(eta=SCENES[name].get("eta", 1e-4), cg_residual_reset_period=period)
    eng.upload(p.copy(), _opts(engine, name, **kw))
    o = oracle.Oracle(p.copy(), _opts(oracle, name, **kw))
    ok_o, cost_o = o.linearize()
    ok_g, cost_g = eng.linearize()
    assert ok_o and ok_g
    assert abs(cost_g - cost_o) <= 1e-12 * cost_o
    its = []
    for radius in (1e4, 1e2):
        assert o.prepare_linear_system(radius) and eng.prepare_linear_system(radius)
        ok_o, it_o, mcc_o = o.solve_linear_system()
        ok_g, it_g, mcc_g = eng.solve_linear_system()
        assert ok_o and ok_g
        assert it_o == it_g, (radius, it_o, it_g)
        its.append(it_g)
        assert abs(mcc_g - mcc_o) <= 1e-9 * abs(mcc_o), radius
        for which, width in STEPS:
            e, k = block_err(eng.read(which), o.read(which), width)
            assert e <= 1e-8, "step %d @%g: block %d, error %.3g" % (which, radius, k, e)
    assert max(its) >= 10, its  # period 10 resets at least once
    o.close()


def test_residual_reset_full_solve(eng, oracle):
    """ITERATIVE_SCHUR with a reset every second CG iteration: the oracle's trajectory."""
    p0 = synthetic.make_scene(**SCENES["pinhole_shared"]["scene"])
    po, pg = p0.copy(), p0.copy()
    so = oracle.solve(po, _opts(oracle, "pinhole_shared", cg_residual_reset_period=2, max_num_iterations=10))
    sg = eng.solve(pg, _opts(engine, "pinhole_shared", cg_residual_reset_period=2, max_num_iterations=10))
    assert sg.rc == 0 and sg.success and so.success
    assert sg.num_iterations == so.num_iterations and sg.termination_type == so.termination_type, (sg.message, so.message)
    its = [i["linear_solver_iterations"] for i in sg.iterations]
    assert its == [i["linear_solver_iterations"] for i in so.iterations]
    assert max(its) >= 2, its
    assert np.all(np.abs(sg.costs - so.costs) <= 1e-9 * so.costs)
