"""CPU tier of the per-element bounds of tests/precise_gauge.py: the host twin of the gauge force, the link update, the
momentum action and the plaquette (the library's site code compiled for the CPU) on adversarial links, momenta,
spectra and lattice shapes, and negative controls: wrong outputs, made by perturbing the twin's results, that the flat
checks of tests/test_twin_gauge.py accept and the bounds must reject."""
import numpy as np
import pytest
import scipy.linalg

import gauge_cases as G
import precise as PR
import precise_gauge as PG
import precise_gauge_cases as C
from gauge_twin import gauge_twin


@pytest.fixture(scope="module")
def tier():
    return G.Runner(gauge_twin(), "twin")


@pytest.mark.parametrize("links", C.LINKS)
@pytest.mark.parametrize("prec", [8, 4])
@pytest.mark.parametrize("shape", list(C.SHAPES))
def test_force_links(tier, shape, prec, links):
    C.check_force(tier, C.SHAPES[shape], prec, links, "gauss", "plaq+rect", C.EB3["pos"])


@pytest.mark.parametrize("eb3", list(C.EB3))
@pytest.mark.parametrize("prec", [8, 4])
@pytest.mark.parametrize("paths", C.PATHS)
def test_force_paths(tier, paths, prec, eb3):
    X = C.SHAPES["6x2x4x6"] if paths == "table-limit" else C.SHAPES["4x6x8x10"]
    C.check_force(tier, X, prec, "mixed", "spread", paths, C.EB3[eb3], antiperiodic=True)


@pytest.mark.parametrize("antiperiodic", [False, True])
@pytest.mark.parametrize("links", C.LINKS)
@pytest.mark.parametrize("prec", [8, 4])
@pytest.mark.parametrize("mom", C.MOMS)
def test_force_moms(tier, mom, prec, links, antiperiodic):
    C.check_force(tier, C.SHAPES["2x4x6x4"], prec, links, mom, "symanzik48", C.EB3["neg"], antiperiodic)


UPDATE_RUNS = [(0.7, False), (0.7, True), (-0.4, False)]  # (dt, conj_mom)


@pytest.mark.parametrize("run", range(len(UPDATE_RUNS)))
@pytest.mark.parametrize("prec", [8, 4])
@pytest.mark.parametrize("kind", C.SPECTRA)
def test_update(tier, kind, prec, run):
    dt, conj = UPDATE_RUNS[run]
    X = C.SHAPES["6x2x4x6"]
    C.check_update(tier, X, prec, kind, dt, conj, exact=True)
    if kind in C.SMALL:
        C.check_update(tier, X, prec, kind, dt, conj, exact=False)


@pytest.mark.parametrize("prec", [8, 4])
@pytest.mark.parametrize("shape", list(C.SUM_SHAPES))
def test_sums(tier, shape, prec):
    X = C.SUM_SHAPES[shape]
    i = list(C.SUM_SHAPES).index(shape)
    C.check_mom_action(tier, X, prec, C.MOMS[i % len(C.MOMS)])
    C.check_plaquette(tier, X, prec, C.LINKS[i % len(C.LINKS)])


def test_reference_exponential_cross_checks():
    """the long-double closed form against the long-double Taylor series with scaling and squaring, and both against
    scipy.linalg.expm, on every spectrum"""
    X = C.SHAPES["6x2x4x6"]
    for kind in C.SPECTRA:
        mom = C.spectrum_mom(X, kind, 0.7, 8)
        P, _ = PG.traceless(mom, 8)
        A = np.longdouble(0.7) * P
        Q = -1j * A
        c0, c1 = PG.invariants(Q)
        ok = c1 >= 1e-3
        taylor = PG.expm_taylor(A)
        if ok.any():
            closed = PG.assemble(PG.exp_coeffs(c0[ok], c1[ok]), Q[ok])
            n = np.abs(A[ok]).astype(np.float64).max((-2, -1))
            assert np.all(np.abs(closed - taylor[ok]).astype(np.float64).max((-2, -1)) <= 1e-17 * np.maximum(1, n)), kind
        A64 = A.astype(np.complex128).reshape(-1, 3, 3)
        sp = np.array([scipy.linalg.expm(a) for a in A64])
        ref = PG.expm(A).astype(np.complex128).reshape(-1, 3, 3)
        assert np.abs(sp - ref).max() <= 1e-13, kind


# ---------------------------------------------------------------------------------------------- negative controls
def rejected(got, res, prec, what):
    r = PR.ratio(got, res, prec)
    print(f"{what}: max err/bound = {r:.3g} (must be > 1)")
    assert r > 1, f"{what}: a wrong output passed the check (max err/bound {r:.3g})"
    return r


def window_perturbation(err_now, lo, hi, where):
    """the perturbation sqrt(lo hi) at the elements `where` whose window hi / lo is at least 10 (a wrong value inside
    (lo, hi) passes the flat check and fails the bound), with the sign of the error already there"""
    width = np.where(where, hi / lo, 0)
    sel = width >= 10
    print(f"window: widest {width.max():.3g}x, {int(sel.sum())} elements at >= 10x")
    assert sel.any(), "no element with a window of at least 10x"
    return np.where(sel, np.where(err_now < 0, -1, 1) * np.sqrt(lo * hi), 0)


def _no_pad(mom):
    return np.nan_to_num(np.asarray(mom, np.float64))


def test_rejects_fp32_force_error_in_the_smooth_block(tier):
    """an error at the links of the eps = 1e-6 block of the mixed field: the flat check divides by the largest force,
    which is in the Haar part"""
    X, prec = C.SHAPES["4x6x8x10"], 4
    p, c = G.path_set("plaq+rect")
    got, res, _ = C.check_force(tier, X, prec, "mixed", "zero-parity", "plaq+rect", C.EB3["pos"])
    gauge = C.links(X, "mixed").astype(np.float32)
    mom0 = _no_pad(C.mom_field(X, "zero-parity", prec))
    want = G.force(mom0, gauge, X, p, c, float(np.float32(C.EB3["pos"])))
    g = got.astype(np.float64)[..., :9]
    hi = 1e-5 * np.abs(want - mom0)[..., :9].max() - np.abs(g - want[..., :9]).max()
    lo = PR.out_bound(PR.Result(res.ref[..., :9], res.bound[..., :9]), prec).astype(np.float64)
    smooth = np.broadcast_to(C.smooth_sites(X)[:, None, None], lo.shape)
    bad = g + window_perturbation((g - res.ref[..., :9]).astype(np.float64), lo, hi, smooth)
    assert G.deviation(bad, want[..., :9], mom0[..., :9]) <= 1e-5, "the flat check should accept this output"
    rejected(bad, PR.Result(res.ref[..., :9], res.bound[..., :9]), prec, "fp32 force error in the smooth block")


def test_rejects_fp64_update_error_at_large_momenta(tier):
    """an error at the links with |dt P| >= 20, where the flat threshold 1e-14 |dt P|^2 exceeds the linear bound"""
    X, prec, dt = C.SHAPES["6x2x4x6"], 8, 0.7
    got, res, _, gauge, mom = C.check_update(tier, X, prec, "large", dt)
    P = G.traceless_p(_no_pad(mom))
    Uc = G.cplx(gauge)
    want = G.to_qdp(np.array([[scipy.linalg.expm(dt * P[v, mu]) for v in range(P.shape[0])] for mu in range(4)]) @ Uc)
    thr = 1e-14 * max(1.0, np.abs(dt * P).max() ** 2)
    hi = thr - np.abs(got - want).max()
    lo = PR.out_bound(res, prec).astype(np.float64)
    big = np.linalg.norm(dt * P, 2, axis=(-2, -1)).T >= 20          # [4][V]
    where = np.broadcast_to(big[..., None, None, None], lo.shape)
    bad = got + window_perturbation((got - res.ref).astype(np.float64), lo, hi, where)
    assert np.abs(bad - want).max() <= thr, "the flat check should accept this output"
    rejected(bad, res, prec, "fp64 update error at |dt P| >= 20")


def test_rejects_fp32_mom_action_site_sums(tier):
    """each site's four-link sum accumulated in fp32 instead of double"""
    X, prec = C.SHAPES["4x6x8x10"], 4
    S, res, _, mom = C.check_mom_action(tier, X, prec, "gauss")
    m = mom.astype(np.float64)[..., :9]
    link = (m[..., :6] ** 2).sum(-1) + 0.5 * (m[..., 6:9] ** 2).sum(-1) - 4.0   # [V][4]
    site = np.zeros(link.shape[0], np.float32)
    for mu in range(4):
        site = (site + link[:, mu].astype(np.float32)).astype(np.float32)
    bad = float(site.astype(np.float64).sum())
    assert abs(bad - G.mom_action(_no_pad(mom)[..., :10])) <= 1e-7 * np.abs(m).sum(), "the flat check should accept it"
    rejected(np.array([bad]), res, 8, "fp32 site sums of the momentum action")


def test_rejects_a_write_of_the_mom_pad(tier):
    """the force writing mom[..., 9] (zero): the flat check compares the pad with the restatement's zero pad, the bound
    does not look at it, the bit check does"""
    X, prec = C.SHAPES["4x6x8x10"], 8
    p, c = G.path_set("plaq")
    got, res, _ = C.check_force(tier, X, prec, "haar", "gauss", "plaq", C.EB3["pos"])
    mom0 = C.mom_field(X, "gauss", prec)
    bad = got.copy()
    bad[..., 9] = 0.0
    want = G.force(_no_pad(mom0), C.links(X, "haar"), X, p, c, C.EB3["pos"])
    assert G.deviation(bad, want, _no_pad(mom0)) <= 1e-13, "the flat check should accept this output"
    assert PR.ratio(bad[..., :9], PR.Result(res.ref[..., :9], res.bound[..., :9]), prec) <= 1
    assert not C.same_bits(bad[..., 9], mom0[..., 9]), "a write of the pad passed the bit check"


def test_rejects_a_sign_error_in_the_smooth_block(tier):
    """the force of the smooth block's links with the opposite sign, fp32: there it is about 1e-6 of the Haar part's, so
    the flat check (relative to the largest force) accepts it"""
    X, prec = C.SHAPES["4x6x8x10"], 4
    p, c = G.path_set("plaq")
    got, res, _ = C.check_force(tier, X, prec, "mixed", "zero-parity", "plaq", C.EB3["pos"])
    mom0 = _no_pad(C.mom_field(X, "zero-parity", prec))
    want = G.force(mom0, C.links(X, "mixed").astype(np.float32), X, p, c, float(np.float32(C.EB3["pos"])))
    # the links whose momentum was zero and whose plaquettes all lie inside the smooth block (1 <= t <= X[3] / 2 - 2)
    # carry the smooth force alone: flip it there
    t = np.concatenate([C.F.cb_coords(X, q)[:, 3] for q in range(2)])
    inner = (t >= 1) & (t <= X[3] // 2 - 2) & (np.arange(len(mom0)) < len(mom0) // 2)
    # and whose flipped force stays below the flat threshold, 1e-5 of the largest force
    fmax = np.abs(want - mom0)[..., :9].max()
    flip = inner[:, None] & (np.abs(got[..., :9]).max(-1) <= 0.4e-5 * fmax)
    assert flip.sum() >= 2 * inner.sum(), "most links of the smooth block should be flipped"
    bad = got.copy()
    bad[flip, :9] = -bad[flip, :9]
    assert G.deviation(bad[..., :9], want[..., :9], mom0[..., :9]) <= 1e-5, "the flat check should accept this output"
    rejected(bad[..., :9], PR.Result(res.ref[..., :9], res.bound[..., :9]), prec, "sign error in the smooth block")
