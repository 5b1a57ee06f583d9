"""CPU tier of gauge smearing, on the host twin (tests/smeartwin), which runs the site code and the launch sequence of
inst_gauge_smear.cu: against the numpy restatement tests/smear_ref.py for every kind and ignored direction, stout against
the gauge force plus the link update, the identity at zero coefficients, SU(3) output, the ignored direction and time
slices, constant abelian flux as a fixed point, gauge covariance and the boundary sign, the projection on crafted
matrices, negative controls that each check must reject, and the argument checks."""
import ctypes as C

import numpy as np
import pytest

import flow_cases as FC
import flow_ref as FR
import gauge_cases as GC
import smear_cases as SC
import smear_ref as SR
from quda_b200 import gauge as GP
from smear_twin import smear_twin

twin = SC.twin


def ref(gauge, X, kind, ign, n_steps=SC.STEPS, control=None, coeffs=None):
    return SR.smear(gauge, X, kind, n_steps, ign, control, **(coeffs or SC.COEFFS[kind]))


# ------------------------------------------------------------------ 1. the restatement; SU(3); the ignored direction
@pytest.mark.parametrize("X", SC.SHAPES)
@pytest.mark.parametrize("kind", SC.KINDS)
@pytest.mark.parametrize("ign", SC.IGNORE)
@pytest.mark.parametrize("field", sorted(SC.FIELDS))
def test_twin_matches_restatement(X, kind, ign, field):
    gauge = SC.FIELDS[field](X, 7)
    got = twin().smear(gauge, X, kind, dir_ignore=ign)
    assert np.abs(got - ref(gauge, X, kind, ign)).max() <= 1e-12
    assert max(SC.su3_deviation(got)) <= 1e-13
    if ign >= 0:
        assert np.array_equal(got[ign], gauge[ign])
    got4 = twin().smear(gauge, X, kind, dir_ignore=ign, prec=4)
    assert np.abs(got4 - got).max() <= 1e-5
    if ign >= 0:
        assert np.array_equal(got4[ign], gauge[ign].astype(np.float32))


# ------------------------------------------------------------------ 2. n calls of one step; in place
@pytest.mark.parametrize("kind", SC.KINDS)
@pytest.mark.parametrize("ign", [-1, 3])
def test_steps_compose_and_in_place(kind, ign):
    X = (6, 2, 4, 6)
    gauge = GC.haar_links(X, 3)
    got = twin().smear(gauge, X, kind, dir_ignore=ign)
    step = gauge
    for _ in range(SC.STEPS):
        step = twin().smear(step, X, kind, n_steps=1, dir_ignore=ign)
    assert np.array_equal(step, got)
    for n in (1, 2, 3):  # the ping-pong ends in either field
        assert np.array_equal(twin().smear(gauge, X, kind, n_steps=n, dir_ignore=ign, in_place=True),
                              twin().smear(gauge, X, kind, n_steps=n, dir_ignore=ign))
    assert np.array_equal(twin().smear(gauge, X, kind, dir_ignore=ign), got)


# ------------------------------------------------------------------ 3. stout = gauge force + link update
@pytest.mark.parametrize("X", [(4, 6, 8, 10), (6, 2, 4, 6)])
@pytest.mark.parametrize("field", sorted(SC.FIELDS))
def test_stout_is_force_plus_update(X, field):
    gauge = SC.FIELDS[field](X, 5)
    rho = SC.COEFFS["stout"]["rho"]
    V = int(np.prod(X))
    r = twin()
    paths, coeffs = GP.FLOW_ACTIONS["wilson"]
    mom = r.force(np.zeros((V, 4, 10)), gauge, X, paths, coeffs, rho)
    want = r.update(gauge, mom, X, 1.0, exact=True)
    got = r.smear(gauge, X, "stout", n_steps=1, dir_ignore=-1)
    assert np.array_equal(got, want)  # the same path walk, projection and exponential, in the same order
    # and the Euler step of the Wilson flow of the restatement, 0.1 apart from its RK3 step
    assert np.abs(got - FR.flow(gauge, X, paths, coeffs, rho, 1, step=FR.euler_step)).max() <= 1e-12


# ------------------------------------------------------------------ 4. zero coefficients
@pytest.mark.parametrize("kind", SC.KINDS)
@pytest.mark.parametrize("ign", SC.IGNORE)
def test_zero_coefficients_return_the_input(kind, ign):
    X = (4, 6, 8, 10)
    gauge = GC.haar_links(X, 4)
    zero = {n: 0.0 for n in GP.SMEAR_KINDS[kind][1]}
    if kind == "ovrimp_stout":
        zero["epsilon"] = -0.25
    for prec in (8, 4):
        got = twin().smear(gauge, X, kind, dir_ignore=ign, prec=prec, coeffs=zero)
        assert np.array_equal(got, gauge.astype(got.dtype))


# ------------------------------------------------------------------ 6. locality in time with t ignored
@pytest.mark.parametrize("kind", SC.KINDS)
def test_t_ignored_keeps_time_slices_apart(kind):
    X = (4, 6, 4, 6)
    gauge = GC.haar_links(X, 6)
    other = np.array(gauge)
    sl = SC.time_slice_sites(X, 2)
    other[:, sl] = GC.haar_links(X, 7)[:, sl]
    a = twin().smear(gauge, X, kind, dir_ignore=3)
    b = twin().smear(other, X, kind, dir_ignore=3)
    rest = np.setdiff1d(np.arange(int(np.prod(X))), sl)
    assert np.array_equal(a[:, rest], b[:, rest])
    assert np.abs(a[:, sl] - b[:, sl]).max() > 0.1


# ------------------------------------------------------------------ 7. constant abelian flux is a fixed point
@pytest.mark.parametrize("kind", SC.KINDS)
@pytest.mark.parametrize("ign", SC.IGNORE)
def test_constant_abelian_flux_is_a_fixed_point(kind, ign):
    X = (4, 6, 8, 10)
    planes, _ = FC.flux_cases()[0]
    gauge, _ = FR.abelian_flux(X, planes)
    got = twin().smear(gauge, X, kind, dir_ignore=ign)
    assert np.abs(got - gauge).max() <= 1e-13
    e, q, _ = twin().observables(gauge, X)
    e2, q2, _ = twin().observables(got, X)
    assert np.abs(np.subtract(e2, e)).max() <= 1e-13 and abs(q2 - q) <= 1e-13


# ------------------------------------------------------------------ 8. gauge covariance, boundary sign
@pytest.mark.parametrize("kind", SC.KINDS)
@pytest.mark.parametrize("ign", [-1, 3])
def test_gauge_covariance_and_boundary_sign(kind, ign):
    X = (4, 6, 8, 10)
    gauge = GC.haar_links(X, 8)
    g = FR.random_su3((X[3], X[2], X[1], X[0]), 9)
    f = twin().smear(gauge, X, kind, dir_ignore=ign)
    f2 = twin().smear(FR.gauge_transform(gauge, X, g), X, kind, dir_ignore=ign)
    assert np.abs(f2 - FR.gauge_transform(f, X, g)).max() <= 1e-12
    p, p2 = twin().plaquette(f, X), twin().plaquette(f2, X)
    assert np.abs(np.subtract(p2, p)).max() <= 1e-12
    fa = twin().smear(GC.antiperiodic(gauge, X), X, kind, dir_ignore=ign)
    assert np.array_equal(fa, GC.antiperiodic(f, X))


# ------------------------------------------------------------------ 9. the projection on crafted matrices
def project(w, prec=8):
    w = np.ascontiguousarray(GC.to_qdp(np.asarray(w, dtype=np.complex128)), dtype=np.float64 if prec == 8 else np.float32)
    p = np.zeros_like(w)
    assert smear_twin().twin_su3_project(p.ctypes.data, w.ctypes.data, len(w), prec) == 0
    return GC.cplx(p)


def _with_det_phase(phi, seed):
    """a unitary matrix with determinant e^{i phi}, times a positive Hermitian factor"""
    u = FR.random_su3((), seed) @ np.diag([np.exp(1j * phi), 1, 1])
    h = np.diag([2.0, 0.7, 1.3])
    return u @ h


def test_projection_on_crafted_matrices():
    cases = {
        "minus identity (phase pi)": -np.eye(3, dtype=complex),
        "exchange (det exactly -1)": np.eye(3, dtype=complex)[[1, 0, 2]] * 1.5,
        "diag(-1, i, -i)": np.diag([-1, 1j, -1j]) @ np.diag([2.0, 0.5, 1.0]),
        "phase pi - 1e-12": _with_det_phase(np.pi - 1e-12, 2),
        "phase -pi + 1e-12": _with_det_phase(-np.pi + 1e-12, 3),
        "negative real det": np.diag([-2.0, 1.0, 0.5]).astype(complex),
        "negative real det, real entries": np.array([[0.5, -1.0, 0.25], [2.0, 0.5, -0.5], [0.0, 1.0, 1.5]]) @ np.diag([-1, 1, 1]),
        "singular value 1e-6": FR.random_su3((), 6) @ np.diag([1.0, 1e-6, 0.8]) @ FR.random_su3((), 7),
        "identity": np.eye(3, dtype=complex),
    }
    W = np.stack(list(cases.values()))
    got, want = project(W), SR.project(W)
    # the near-singular case: the first Newton step inverts a matrix of condition 1e6 by cofactors (as the reference's
    # iteration does), which leaves an error of a few 1e-8 in the polar factor; the SVD restatement itself moves by 1e-10
    # under a 1e-16 perturbation of this input
    tol = {"singular value 1e-6": 1e-7}
    for name, g, w in zip(cases, got, want):
        print(f"{name:32s} |P - ref| {np.abs(g - w).max():.2e}  det {np.linalg.det(g):.15f}")
        assert np.abs(g - w).max() <= tol.get(name, 1e-12), name
        assert abs(np.linalg.det(g) - 1) <= 1e-13 and np.abs(g.conj().T @ g - np.eye(3)).max() <= 1e-13, name
    # the branch: at pi and just below it the cube root is e^{i pi/3}, just above -pi it is e^{-i pi/3}
    for k in (0, 1, 2):  # the exact phase pi and pi - 1e-12 take e^{i pi/3} (times a positive matrix, the polar factor)
        u, _, vh = np.linalg.svd(W[k])
        assert np.abs(got[k] @ np.linalg.inv(u @ vh) - np.exp(-1j * np.pi / 3) * np.eye(3)).max() <= 2e-12
    u, _, vh = np.linalg.svd(W[4])  # -pi + 1e-12 takes e^{-i pi/3}
    assert np.abs(got[4] @ np.linalg.inv(u @ vh) - np.exp(1j * np.pi / 3) * np.eye(3)).max() <= 2e-12
    # fp32 where the branch and the conditioning are resolved at its precision (the phases pi -+ 1e-12 round onto pi)
    keep = [k for k, name in enumerate(cases) if "1e-12" not in name and "1e-6" not in name]
    assert np.abs(project(W[keep], prec=4) - want[keep]).max() <= 1e-5


# ------------------------------------------------------------------ 10. negative controls
def test_projecting_the_link_sum_fails_the_sign_check():
    X = (4, 6, 8, 10)
    gauge = GC.haar_links(X, 13)
    ctl = {"sum_projection": True}
    f = ref(gauge, X, "ape", -1, 1, ctl)
    fa = ref(GC.antiperiodic(gauge, X), X, "ape", -1, 1, ctl)
    assert np.abs(fa - GC.antiperiodic(f, X)).max() > 0.1
    f = ref(gauge, X, "ape", -1, 1)  # the product with U^+ passes
    assert np.abs(ref(GC.antiperiodic(gauge, X), X, "ape", -1, 1) - GC.antiperiodic(f, X)).max() <= 1e-13


def test_ape_normalised_by_four_fails_the_restatement_check():
    X = (4, 4, 4, 4)
    gauge = GC.near_identity_links(X, 7, 0.1)
    got = twin().smear(gauge, X, "ape", dir_ignore=-1)
    assert np.abs(got - ref(gauge, X, "ape", -1, control={"ape_norm": 4})).max() > 1e-4


def test_wrong_level2_link_fails_the_restatement_check():
    X = (4, 4, 4, 4)
    gauge = GC.haar_links(X, 7)
    got = twin().smear(gauge, X, "hyp", dir_ignore=-1)
    assert np.abs(got - ref(gauge, X, "hyp", -1, control={"wrong_level2": True})).max() > 1e-3


# ------------------------------------------------------------------ 11. validation
def test_refusals():
    X = (4, 4, 4, 4)
    V = int(np.prod(X))
    r = twin()
    g = GC.haar_links(X, 1)
    for type_, coeff, ign, n in ((4, [0.1], -1, 1), (-1, [0.1], -1, 1), (0, [np.nan], -1, 1), (1, [np.inf], 3, 1),
                                 (2, [0.1, np.nan], -1, 1), (3, [0.1, 0.2, np.inf], -1, 1), (0, [0.1], -2, 1),
                                 (0, [0.1], 5, 1), (0, [0.1], -1, 0), (3, [0.1, 0.1, 0.1], 2, -1)):
        assert r.smear_rc(g, X, type_, coeff, ign, n)[0] == -1
    # coefficients a kind does not use are not read
    assert r.smear_rc(g, X, 0, [0.1, np.nan, np.nan], -1, 1)[0] == 0
    assert r.smear_rc(g, X, 3, [0.1, 0.1, 0.1], 4, 1)[0] == 0
    lib = smear_twin()
    buf = np.zeros((4, V, 18))
    q = (C.c_void_p * 4)(*[buf[d].ctypes.data for d in range(4)])
    qn = (C.c_void_p * 4)(buf[0].ctypes.data, None, buf[2].ctypes.data, buf[3].ctypes.data)
    Xc = (C.c_int * 4)(*X)
    c = (C.c_double * 3)(0.1, 0.1, 0.1)
    for out, inp, cc in ((None, q, c), (q, None, c), (qn, q, c), (q, qn, c), (q, q, None)):
        assert lib.twin_gauge_smear(out, inp, Xc, 8, 0, cc, -1, 1, None) == -1
    assert lib.twin_gauge_smear(q, q, (C.c_int * 4)(4, 4, 4, 3), 8, 0, c, -1, 1, None) == -1
    assert lib.twin_gauge_smear(q, q, Xc, 2, 0, c, -1, 1, None) == -1
    assert "dir_ignore" in (lib.twin_gauge_smear(q, q, Xc, 8, 0, c, 7, 1, None), lib.twin_last_error().decode())[1]
