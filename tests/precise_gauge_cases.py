"""Cases for the per-element bounds of tests/precise_gauge.py, shared by the CPU tier (the host twin, tests/gaugetwin) and
the GPU tier (libquda_b200.so): one body per check, run on a gauge_cases.Runner."""
import numpy as np

import clover_force_ref as CF
import gauge_cases as G
import precise as PR
import precise_clover_cases as PCC
import precise_gauge as PG
from quda_b200 import fields as F
from quda_b200 import lib as L

SHAPES = PCC.SHAPES
# the sums only: 512 CTA partials per parity, and 135 (a ragged second stage)
SUM_SHAPES = {**SHAPES, "16^3x32": (16, 16, 16, 32), "6x6x30x32": (6, 6, 30, 32)}
LINKS = ["haar", "eps1e-2", "eps1e-5", "mixed"]
MOMS = ["gauss", "spread", "zero-parity"]
EB3 = {"pos": 0.2, "neg": -0.35, "tiny": 1e-7}
PATHS = ["plaq", "plaq+rect", "symanzik48", "table-limit"]


# ---------------------------------------------------------------------------------------------- fields
def links(X, kind, seed=11, antiperiodic=False):
    """QDP links [4][V][3][3][2]: Haar, exp(i eps H), or 'mixed': Haar with an eps = 1e-6 block of the first half of the
    time slices, so that the force varies by about 10^6 inside one field"""
    if kind == "haar":
        g = G.haar_links(X, seed)
    elif kind.startswith("eps"):
        g = G.near_identity_links(X, seed, float(kind[3:]))
    else:
        g = G.haar_links(X, seed)
        smooth = G.near_identity_links(X, seed + 1, 1e-6)
        blk = smooth_sites(X)
        g[:, blk] = smooth[:, blk]
    return G.antiperiodic(g, X) if antiperiodic else g


def smooth_sites(X):
    """sites (parity-major) of the smooth block of the mixed field: t < X[3] / 2"""
    t = np.concatenate([F.cb_coords(X, p)[:, 3] for p in range(2)])
    return t < X[3] // 2


def mom_field(X, kind, prec, seed=5, scale=0.1):
    """momenta [V][4][10] with the NaN sentinel in the pad: Gaussian, octave-spread (each link x 2^k, k in [-20, 10] for
    fp64, [-10, 5] for fp32) or Gaussian with parity 0 zero"""
    V = int(np.prod(X))
    m = G.random_mom(V, seed, scale)
    rng = np.random.default_rng(seed + 1)
    if kind == "spread":
        lo, hi = (-20, 10) if prec == 8 else (-10, 5)
        m *= np.exp2(rng.integers(lo, hi + 1, (V, 4)))[..., None]
    elif kind == "zero-parity":
        m[:V // 2] = 0
    m[..., 9] = np.nan
    return m.astype(PG.field_t(prec))


def path_set(name):
    """(paths, coefficients): gauge_cases.path_set, or 'table-limit': B200_GAUGE_MAX_PATHS 5x1 rectangles per direction
    (the longest path a row holds) with alternating signs"""
    if name != "table-limit":
        return G.path_set(name)
    k = L.GAUGE_MAX_LENGTH // 2 - 2
    loops = [[[mu + 1] * (1 + k) + [s * ((mu + 1) % 4 + 1)] + [-(mu + 1)] * (1 + k) + [-s * ((mu + 1) % 4 + 1)]
              for s in (1, -1)] * (L.GAUGE_MAX_PATHS // 2) for mu in range(4)]
    return G._paths(loops), [(-1) ** i * (1.0 + i / 64) / 16 for i in range(L.GAUGE_MAX_PATHS)]


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


# ---------------------------------------------------------------------------------------------- force
def run_force(runner, gauge, mom, X, paths, coeffs, eb3, prec):
    from quda_b200 import gauge as GP
    table, lengths, n, max_length = GP.path_table(paths)
    if table.shape[2] < max_length:
        table = np.pad(table, ((0, 0), (0, 0), (0, max_length - table.shape[2])))
    rc, got = runner.force_rc(mom, gauge, X, table, lengths, coeffs, n, max_length, eb3, prec)
    runner.check(rc)
    return got


def check_force(runner, X, prec, links_kind, mom_kind, paths, eb3, antiperiodic=False, what=""):
    """mom after one call against its bound, per link and real component; the pad bit-identical; returns (got, res)"""
    gauge = links(X, links_kind, antiperiodic=antiperiodic).astype(PG.field_t(prec))
    mom = mom_field(X, mom_kind, prec)
    p, c = path_set(paths)
    got = run_force(runner, gauge, mom, X, p, c, eb3, prec)
    res = PG.force(gauge, mom, X, p, c, eb3, prec)
    tag = f"force {what}{X} prec={prec} {links_kind}{' antiperiodic' if antiperiodic else ''} {mom_kind} {paths} eb3={eb3}"
    r = PR.assert_within(got[..., :9], PR.Result(res.ref[..., :9], res.bound[..., :9]), prec, tag)
    assert same_bits(got[..., 9], mom[..., 9]), "the pad of mom was written"
    return got, res, r


# ---------------------------------------------------------------------------------------------- update
C1_TARGETS = {"c1-0.5x": 0.5, "c1-0.99x": 0.99, "c1-1.01x": 1.01, "c1-2x": 2.0}
W_TARGETS = {"w-0.5x": 0.5, "w-1x": 1.0, "w-2x": 2.0}
SPECTRA = ["zero", "tiny", *C1_TARGETS, "generic", "large", "degenerate", "degenerate-rot", *W_TARGETS, "c0-zero",
           "c0-max", "c0-min"]
SMALL = {"zero", "tiny", *C1_TARGETS, "generic", "degenerate", *W_TARGETS, "c0-zero", "c0-max", "c0-min"}  # |dt P| <= 1


def _from_eigen(ev, rng):
    """mom [..][10] of P = i q diag(ev) q^+ for random unitary q"""
    z = rng.normal(size=ev.shape + (3,)) + 1j * rng.normal(size=ev.shape + (3,))
    q, _ = np.linalg.qr(z)
    return CF.mom_from_matrices(np.einsum("...ij,...j,...kj->...ik", q, 1j * ev, q.conj()))


def spectrum_mom(X, kind, dt, prec, seed=22):
    """momenta [V][4][10] (pad NaN) whose dt P has the spectrum `kind`: c1 of dt P at a multiple of kExpSeriesC1, w =
    Im of the split of the two nearest eigenvalues at a multiple of 0.05 (the sin w / w series threshold), c0 = 0 or
    +-c0_max (two equal eigenvalues, the r > 1 clamp), degenerate exactly (diagonal) or after a rotation"""
    V = int(np.prod(X))
    rng = np.random.default_rng(seed)
    shp = (V, 4)
    if kind == "zero":
        m = np.zeros(shp + (10,))
    elif kind == "tiny":
        m = G.random_mom(V, seed, 1e-9)
    elif kind == "generic":
        m = G.random_mom(V, seed, 0.3 / abs(dt))
    elif kind == "large":
        m = G.random_mom(V, seed, 1.0)
        n = np.linalg.norm(CF.mom_to_matrices(m), 2, axis=(-2, -1))
        m *= (rng.uniform(1.0, 50.0, shp) / n)[..., None] / abs(dt)
    elif kind in C1_TARGETS:
        m = G.random_mom(V, seed, 1.0)
        Pm = CF.mom_to_matrices(m)
        c1 = -np.einsum("...ij,...ji->...", Pm, Pm).real / 2
        m *= np.sqrt(C1_TARGETS[kind] * PG.EXP_SERIES_C1 / c1)[..., None] / abs(dt)
    elif kind in W_TARGETS or kind.startswith("degenerate") or kind.startswith("c0-max") or kind == "c0-min":
        a = rng.uniform(0.1, 0.3, shp) * rng.choice([-1, 1], shp)
        if kind == "c0-max":
            a = np.abs(a)
        if kind == "c0-min":
            a = -np.abs(a)
        w = W_TARGETS.get(kind, 0.0) * 0.05
        ev = np.stack([2 * a, -a + w, -a - w], -1) / dt
        if kind == "degenerate":  # exactly: a diagonal mom with representable entries
            m = np.zeros(shp + (10,))
            m[..., 6:9] = ev.astype(PG.field_t(prec))
            m[..., 8] = -(m[..., 6] + m[..., 7])
        else:
            m = _from_eigen(ev, rng)
    elif kind == "c0-zero":
        a = rng.uniform(-1.0, 1.0, shp)
        m = _from_eigen(np.stack([a, -a, 0 * a], -1) / dt, rng)
    else:
        raise ValueError(kind)
    m = np.array(m)
    m[..., 9] = np.nan
    return m.astype(PG.field_t(prec))


def check_update(runner, X, prec, kind, dt=0.7, conj_mom=False, exact=True, in_place=False, links_kind="haar",
                 what=""):
    gauge = links(X, links_kind, seed=21).astype(PG.field_t(prec))
    mom = spectrum_mom(X, kind, dt, prec)
    got = runner.update(gauge, mom, X, dt, conj_mom, exact, prec, in_place=in_place)
    res = PG.Update(gauge, mom, X, dt, prec, conj_mom, exact).result
    tag = f"update {what}{X} prec={prec} {kind} dt={dt} conj={conj_mom} exact={exact}"
    r = PR.assert_within(got, res, prec, tag)
    return got, res, r, gauge, mom


# ---------------------------------------------------------------------------------------------- sums
def check_mom_action(runner, X, prec, mom_kind="gauss"):
    mom = mom_field(X, mom_kind, prec, scale=1.0)
    S = runner.mom_action(mom, X, prec)
    res = PG.mom_action(mom, X, prec)
    r = PG.assert_scalar(np.array([S]), res, f"mom action {X} prec={prec} {mom_kind}")
    return S, res, r, mom


def check_plaquette(runner, X, prec, links_kind="haar"):
    gauge = links(X, links_kind, seed=31).astype(PG.field_t(prec))
    got = runner.plaquette(gauge, X, prec)
    res = PG.plaquette(gauge, X, prec)
    assert got[0] == 0.5 * (got[1] + got[2])
    r = PG.assert_scalar(np.array(got), res, f"plaquette {X} prec={prec} {links_kind}")
    return got, res, r
