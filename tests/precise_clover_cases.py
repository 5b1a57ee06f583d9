"""Cases for the per-element bounds of tests/precise_clover.py, shared by the CPU tier (the host twins of the clover build
and the clover force) and the GPU tier (libquda_b200.so): one body per check, run on a `Tier`."""
import numpy as np

import clover_build_ref as R
import clover_force_cases as FC
import oracle
import precise as PR
import precise_clover as PCL
from quda_b200 import comm
from quda_b200 import dslash as D
from quda_b200 import fields as F
from quda_b200 import lib as L

COEFF = 0.12195 * 1.7
# links: Haar, near the identity (exp(i eps H)), and t periodic or antiperiodic
LINKS = {"haar": dict(), "eps1e-2": dict(eps=1e-2), "eps1e-5": dict(eps=1e-5, antiperiodic_t=False),
         "haar-periodic": dict(antiperiodic_t=False)}
SHAPES = {"4x6x8x10": (4, 6, 8, 10), "2x4x6x4": (2, 4, 6, 4), "6x4x4x2": (6, 4, 4, 2),
          "6x2x4x6": (6, 2, 4, 6), "4x6x2x10": (4, 6, 2, 10), "8^4": (8, 8, 8, 8)}
# build fields: (links, clover), clover "ill": coeff chosen for kappa_2 = 1e3 on the worst block
BUILD_FIELDS = {"haar": ("haar", "near"), "eps1e-2": ("eps1e-2", "near"), "eps1e-5": ("eps1e-5", "near"),
                "haar-periodic": ("haar-periodic", "near"), "ill": ("haar", "ill")}
MASKS = [tuple((m >> d) & 1 for d in range(4)) for m in range(1, 16)]


class Tier:
    """the twins (gpu False) or libquda_b200.so (gpu True), with the memory each one reads"""

    def __init__(self, gpu):
        self.gpu = gpu
        if gpu:
            import torch
            self.torch = torch
            self.clover_be, self.force_lib, self.prefix = None, L.load(), "b200"
        else:
            from clover_twin import clover_twin
            from force_twin import force_twin
            self.clover_be, self.force_lib, self.prefix = clover_twin(), force_twin(), "twin"

    def put(self, a):
        a = np.ascontiguousarray(a)
        return self.torch.from_numpy(a).cuda() if self.gpu else a.copy()

    def get(self, a):
        return a.cpu().numpy() if self.gpu else a

    def ptr(self, a):
        return a.data_ptr() if self.gpu else a.ctypes.data

    def build(self, gauge, X, prec, coeff, border=(0, 0, 0, 0)):
        """(packed A, A^-1, trlog) of b200_compute_clover + b200_clover_invert_packed"""
        packed = self.put(np.zeros((int(np.prod(X)), 2, 36), oracle._dt(prec)))
        D.compute_clover(packed, self.put(gauge), X, border, prec, coeff, backend=self.clover_be)
        inv = self.put(np.zeros((int(np.prod(X)), 2, 36), oracle._dt(prec)))
        tl = D.clover_invert(inv, packed, X, prec, backend=self.clover_be)
        return self.get(packed), self.get(inv), tl

    def force(self, case, prec, piece="all"):
        return FC.run(self.force_lib, self.prefix, case, piece, prec, to_dev=self.put, to_host=self.get, ptr=self.ptr)


# ---------------------------------------------------------------------------------------------- fields
def gauge_field(X, links, seed, prec):
    return PR.random_gauge(X, seed, **LINKS[links]).astype(oracle._dt(prec))


def ill_coeff(gauge, X, cond=1e3):
    """coeff such that A = 1 + coeff B stays positive definite on every block and reaches kappa_2 = cond on the worst"""
    B = R.unpack(R.compute_clover(np.asarray(gauge, np.float64), X, 1.0)) - np.eye(6)
    w = np.linalg.eigvalsh(B)
    lo, hi = 0.0, -1.0 / w[..., 0].min()
    for _ in range(200):
        c = 0.5 * (lo + hi)
        k = np.max((1 + c * w[..., -1]) / (1 + c * w[..., 0]))
        lo, hi = (c, hi) if k < cond else (lo, c)
    return lo


def coeff_for(gauge, X, clover):
    return ill_coeff(gauge, X) if clover == "ill" else COEFF


def extend_periodic(gauge, X, mask):
    """the depth-1 extended QDP links that comm.extend_gauge gives a rank that is its own neighbour: the periodic wrap
    by one site on both sides of every dimension in `mask`"""
    Xe = [X[d] + 2 * mask[d] for d in range(4)]
    tail = gauge.shape[2:]
    lex = np.empty_like(gauge)
    lex[:, comm._lex_of_sites(X)] = gauge
    lex = lex.reshape((4, X[3], X[2], X[1], X[0]) + tail)
    pad = [(0, 0)] + [(mask[3 - a], mask[3 - a]) for a in range(4)] + [(0, 0)] * len(tail)
    ext = np.pad(lex, pad, mode="wrap").reshape((4, int(np.prod(Xe))) + tail)
    return np.ascontiguousarray(ext[:, comm._lex_of_sites(Xe)]), Xe


# ---------------------------------------------------------------------------------------------- the clover construction
def check_build(tier, X, prec, links, clover="near", seed=11, what=""):
    """A, A^-1 and tr log A against their bounds; returns (packed, inv, trlog, max ratios)"""
    gauge = gauge_field(X, links, seed, prec)
    coeff = coeff_for(gauge, X, clover)
    A, inv, tl = tier.build(gauge, X, prec, coeff)
    tag = f"{what}{X} prec={prec} {links} {clover}"
    r = {"A": PR.assert_within(A, PCL.clover_build(gauge, X, coeff, prec), prec, f"A {tag}")}
    Iv = PCL.Inverse(A, prec)
    if clover == "ill":
        assert Iv.kappa.max() > 300, Iv.kappa.max()
    r["inv"] = PR.assert_within(inv, Iv.result(), prec, f"A^-1 {tag}")
    r["trlog"] = PR.assert_within(np.array(tl), Iv.trlog(X), 8, f"tr log A {tag}")
    return A, inv, tl, r


def check_border(tier, X, prec, seed=13):
    """every nonzero border mask: the interior of the extended build is the unextended build, bit for bit"""
    gauge = gauge_field(X, "haar", seed, prec)
    A0, _, tl0 = tier.build(gauge, X, prec, COEFF)
    PR.assert_within(A0, PCL.clover_build(gauge, X, COEFF, prec), prec, f"A {X} prec={prec} no border")
    for mask in MASKS:
        ext, _ = extend_periodic(gauge, X, mask)
        A, _, tl = tier.build(ext, X, prec, COEFF, border=mask)
        assert np.array_equal(A, A0), f"border {mask}: the interior differs from the unextended build"
        assert tl == tl0, (mask, tl, tl0)
    return A0, tl0


# ---------------------------------------------------------------------------------------------- the clover force
class ForceCase:
    """n spinor pairs of one kind, links, A and mom on lattice X for b200_clover_force_accumulate; the attributes
    clover_force_cases.run reads, plus the decoded values the reference works on"""

    def __init__(self, X, prec, n, kind, links="haar", clover="near", eps_zero=None, seed=7):
        self.X, self.n, self.prec, self.kind = tuple(X), n, prec, kind
        V, Vh = int(np.prod(X)), F.volume_cb(X)
        dt = oracle._dt(prec)
        self.gauge = gauge_field(X, links, seed, prec)
        coeff = coeff_for(self.gauge, X, clover)
        self.packed = R.compute_clover(self.gauge.astype(np.float64), X, coeff).astype(dt)
        spread = 0 if kind != "spread" else (200 if prec == 8 else 30)
        pts = None
        if kind == "points":
            pts = sorted({0, Vh // 3, Vh + 1, V - 1})
        gen = lambda s: PR.gaussian_spinor(X, s, nparity=2, spread=spread, points=pts)  # noqa: E731
        self.xs = [gen(seed + 10 + i) for i in range(n)]
        self.ps = [gen(seed + 100 + i) for i in range(n)]
        rng = np.random.default_rng(seed)
        # spread: no mom, so that the update of the smallest sites is not hidden under the rounding of mom
        scale = 0.0 if kind == "spread" else 0.1
        self.mom = (scale * FC.CF.mom_from_matrices(FC.CF.ta(rng.normal(size=(V, 4, 3, 3))
                                                              + 1j * rng.normal(size=(V, 4, 3, 3))))).astype(dt)
        self.mom[..., 9] = rng.normal(size=(V, 4))  # the pad: must come back untouched
        self.fc = list(rng.uniform(-1.0, 1.0, n))
        self.eps = [tuple(rng.uniform(-0.5, 0.5, 2)) for _ in range(n)]
        if eps_zero is not None:
            self.eps = [tuple(0.0 if p == eps_zero else e[p] for p in range(2)) for e in self.eps]
        # points: no tr[sigma A^-1] term, so that links that touch no nonzero site carry mom alone
        self.sigma_coeff = 0.0 if kind == "points" else 0.5
        self.trlog_parity = 1
        self.support = pts

    def coefficients(self, piece):
        return FC.Case.coefficients(self, piece)

    def native(self, host, prec):
        Vh = F.volume_cb(self.X)
        return np.concatenate([F.spinor_to_native(host[p * Vh:(p + 1) * Vh], prec) for p in range(2)])

    def decoded(self, host):
        """native-basis lexicographic [t][z][y][x][4][3] of exactly what the kernel reads"""
        Vh = F.volume_cb(self.X)
        halves = [PR.decode_spinor(F.spinor_to_native(host[p * Vh:(p + 1) * Vh], self.prec), Vh, self.prec)[0]
                  for p in range(2)]
        return R.to_lex(np.concatenate(halves), self.X)

    def reference(self, piece="all"):
        fc, eps, sc = self.coefficients(piece)
        return PCL.Force(self.gauge, self.packed, [self.decoded(x) for x in self.xs], [self.decoded(p) for p in self.ps],
                         fc, eps, sc, self.trlog_parity, self.mom, self.X, self.prec)


# (shape, kind, n, links, clover, parity with eps = 0): each force case on both tiers, in fp64 and fp32
FORCE_CASES = {
    "4x6x8x10-gauss-n3": ("4x6x8x10", "gauss", 3, "haar", "near", None),
    "4x6x8x10-points-n1": ("4x6x8x10", "points", 1, "haar", "near", None),
    "2x4x6x4-spread-n3": ("2x4x6x4", "spread", 3, "eps1e-2", "near", 0),
    "6x4x4x2-gauss-n1": ("6x4x4x2", "gauss", 1, "haar-periodic", "near", 1),
    "6x2x4x6-spread-n12": ("6x2x4x6", "spread", 12, "haar", "near", None),
    "4x6x2x10-points-n3": ("4x6x2x10", "points", 3, "eps1e-5", "near", None),
    "6x2x4x6-gauss-ill": ("6x2x4x6", "gauss", 3, "haar", "ill", None),
    "8^4-gauss-n12": ("8^4", "gauss", 12, "haar", "near", None),
}


def force_case(name, prec):
    shape, kind, n, links, clover, ez = FORCE_CASES[name]
    return ForceCase(SHAPES[shape], prec, n, kind, links, clover, ez)


def check_force(tier, case, what=""):
    """mom after one call against the reference, per link and real component; returns (mom, reference)"""
    got = tier.force(case, case.prec)
    ref = case.reference()
    PR.assert_within(got, ref.result, case.prec, f"force {what}{case.X} prec={case.prec} {case.kind} n={case.n}")
    assert np.array_equal(got[..., 9], case.mom[..., 9].astype(np.float64)), "the pad of mom was written"
    if case.support is not None:  # links away from the nonzero sites: mom re-projected, no force term at all
        untouched = ref.result.bound[..., 0] <= PCL.gamma(PCL.K_TA, PR.U_P[case.prec]) * 2 * np.abs(case.mom[..., :9]).max()
        assert untouched.sum() > untouched.size // 2, "points: most links should carry no force"
    return got, ref
