"""One Levenberg-Marquardt try's linear algebra, read back from the GPU (plp_ba_debug_try) and held against a high-precision
reference of the same operation.

The solves of test_ba_gpu.py / test_ba_shapes_gpu.py compare the OPTIMUM.  LM repairs a slightly wrong step on its next try, so
a trailing-update tile skipped at a ragged edge of the blocked Cholesky, or a Schur term dropped for one pair of keyframes,
costs a few tries and lands on the same optimum.  Here nothing iterates:
  1. the reduced camera system S, g, bp, chi2 and lambda of the first real try against the Schur complement of the full normal
     equations of tests/ba_numpy.py, eliminated landmark by landmark in long double (tests/ba_system_ref.py);
  2. the step dp by its backward error against the downloaded system itself -- independent of the system's conditioning;
  3. the determinism the design relies on (DESIGN.md section 3.5 "deterministic summation order", section 6 "every rank
     solves the identical system").
The observed errors quoted at the bounds were read on an H100 80GB HBM3 (700 W power limit)."""
import numpy as np
import pytest

import ba_data
import ba_system_ref as ref

pytestmark = pytest.mark.gpu

_BACKGROUND = dict(k=(3, 9))


def _handle(ctx, prob, num_ctas=0):
    from plpslam_b200.ba import LocalBA
    st = prob.struct()
    ba = LocalBA(ctx, st, (len(prob.kf_fixed), len(prob.pt_pos_w), len(prob.line_plucker), len(prob.pt_edge_kf),
                           len(prob.line_edge_kf)), num_ctas=num_ctas)
    ba._keep = (prob, st)
    return ba


def _window(n_free, lines=False, per_kf=6):
    """n_free free + 4 fixed keyframes; a few tracks through every keyframe and through 33 of them, `per_kf` ordinary
    landmarks per keyframe: small enough for the dense full normal equations of the reference."""
    n_kf = n_free + 4
    prob = ba_data.make_ba_shape_problem(
        300 + n_free, n_free, 4,
        points=[dict(n=6, k="all"), dict(n=4, k=min(33, n_kf)), dict(n=3, k=2), dict(n=3, k=3, who="fixed"), dict(n=per_kf * n_kf, **_BACKGROUND)],
        lines=[dict(n=2, k=min(40, n_kf)), dict(n=n_kf, **_BACKGROUND)] if lines else ())
    assert int((prob.kf_fixed == 0).sum()) == n_free and (prob.shape["pt_free_deg"][:6] == n_free).all()
    assert (prob.shape["pt_deg"][6:10] == min(33, n_kf)).all() and (prob.shape["pt_free_deg"][13:16] == 0).all()
    return prob


# ---------------------------------------------------------------------------------------------------------------------
# 1. S, g, chi2, lambda
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("num_ctas", [1, 3, 132], ids=lambda c: f"ctas{c}")
@pytest.mark.parametrize("n_free,lines", [(12, False), (32, False), (33, False), (48, False), (71, False), (12, True), (37, True)],
                         ids=lambda v: f"{v}free" if not isinstance(v, bool) else ("lines" if v else "points"))
def test_reduced_system_equals_schur_complement_of_the_full_normal_equations(ctx, n_free, lines, num_ctas):
    """Every 6 x 6 block of S within tol * max|S|, g within tol * max|g|, chi2 to 1e-12, lambda = 1e-5 max diag(H).
    Points only (analytic Jacobians on both sides): observed at most 4.6e-15 for S and 1.1e-14 for g, on either
    representation and at every CTA count; tol = 1e-13, a decade above.  With lines: the kernels and the reference both take
    central differences with delta = 1e-9, whose rounding noise is ~1e-7 relative: observed 4.9e-8 / 5.0e-8 (2.8e-7 for the
    same kernels under tests/cta_emu), tol = 1e-5."""
    prob = _window(n_free, lines)
    ba = _handle(ctx, prob, num_ctas)
    got = ba.debug_try(n_free)
    ba.close()
    err = ref.check_system(got, prob, n_free, 1e-5 if lines else 1e-13)
    print(f"\nBA-SYSTEM n_free={n_free} lines={lines} ctas={num_ctas} S_err={err[0]:.3e} g_err={err[1]:.3e}")


# ---------------------------------------------------------------------------------------------------------------------
# 2. the step solves the system it was computed from
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_free", [1, 2, 31, 32, 33, 37, 48, 64, 71, 100], ids=lambda n: f"{n}free")
def test_step_solves_the_downloaded_system(ctx, n_free):
    """|(S + lambda I) dp - g|_inf <= bound * n * (|S + lambda I|_inf |dp|_inf + |g|_inf), residual in long double from the
    downloaded S, g, lambda.  <= 32: ba_solve_kernel (block = one keyframe, 4 x 4 register tiles of the trailing update).
    Above: ba_chol.cu, 32 columns per step -- 6 n_free = 198: last block 6 wide; 222: 30 wide; 288, 384: the last block is
    full and only the right-hand-side row lies below it; 426, 600: ragged again, 14 and 19 steps.
    ref.backward_error divides by n (...), so 1e-13 would be the bound of a careful FP64 solver.  Observed: 4.2e-18 at one
    keyframe, falling to 6.7e-20 at 100; the bound is a decade above the maximum."""
    prob = _window(n_free, lines=False, per_kf=40)
    ba = _handle(ctx, prob)
    got = ba.debug_try(n_free)
    ba.close()
    assert np.isfinite(got["dp"]).all() and np.abs(got["dp"]).max() > 1e-4, "no step was taken"
    be = ref.backward_error(ref.dense_from_blocks(got["S"], n_free), got["g"], got["dp"], got["lam"])
    print(f"\nBA-BACKWARD n_free={n_free} backward_error={be:.3e}")
    assert be <= 5e-17, be


# ---------------------------------------------------------------------------------------------------------------------
# 3. determinism
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("num_ctas", [1, 132], ids=lambda c: f"ctas{c}")
def test_shared_memory_path_is_bit_reproducible(ctx, num_ctas):
    """No atomics on values, every S entry owned by one thread, partials reduced in a fixed order: two calls on one handle
    give the same bits.  (Two calls, not a loop: an ordering race that shows once in many runs is not what this looks for.)"""
    prob = _window(32, lines=True, per_kf=20)
    ba = _handle(ctx, prob, num_ctas)
    a, b = ba.debug_try(32), ba.debug_try(32)
    ba.close()
    assert np.array_equal(a["packed"], b["packed"]) and np.array_equal(a["dp"], b["dp"]) and a["lam"] == b["lam"]


def test_dense_path_is_reproducible_to_rounding(ctx):
    """More than 32 free keyframes: every landmark adds its blocks to S in HBM with FP64 atomicAdd, whose order changes from
    run to run, so the sums differ in their last bits -- not bitwise equal, by design; 1e-12 relative to the largest entry."""
    prob = _window(48, lines=True, per_kf=20)
    ba = _handle(ctx, prob)
    a, b = ba.debug_try(48), ba.debug_try(48)
    ba.close()
    assert np.abs(a["packed"] - b["packed"]).max() <= 1e-12 * np.abs(a["packed"]).max()
    assert np.abs(a["dp"] - b["dp"]).max() <= 1e-9 * np.abs(a["dp"]).max()   # the solve amplifies by the condition number
    assert abs(a["lam"] - b["lam"]) <= 1e-12 * a["lam"]
