"""Cases for the per-element error bounds of tests/precise.py, shared by the CPU tier (host twin) and the GPU tier
(libquda_b200.so): build native fields from seeded generators, decode exactly what the kernel reads, run one operator
and compare every element of its output with the high-precision reference."""
import numpy as np

import oracle
import ops
import precise as PR
from quda_b200 import dslash as D
from quda_b200 import fields as F


class Fields:
    """Gauge (+ clover) field of one (precision, recon) on the device (or host-twin) memory `mem`, with the decoded
    images the reference works on."""

    def __init__(self, X, prec, recon, mem, seed=1, eps=None, anisotropy=1.0, antiperiodic_t=True, clover=None,
                 compressed=True, dynamic=True):
        self.X, self.prec, self.recon, self.mem = [int(v) for v in X], prec, recon, mem
        self.Vh = F.volume_cb(X)
        tb = -1 if antiperiodic_t else 1
        self.gauge = PR.random_gauge(X, seed, eps, anisotropy, antiperiodic_t)
        gbuf, gmeta = F.gauge_to_native(self.gauge, X, prec, recon)
        self.U = D.GaugeField(mem.put(gbuf), X, prec, recon, gmeta, anisotropy=anisotropy, t_boundary=tb)
        self.G = PR.decode_gauge(gbuf, X, prec, recon, gmeta, anisotropy, tb)
        self.dynamic = dynamic
        if clover is not None:
            host = oracle.random_clover(X, 8, seed=seed + 1) if clover == "near" else PR.hpd_clover(X, seed + 1, clover)
            self.clover = host
            cbuf, cmeta = F.clover_to_native(host, X, prec, compressed=compressed)
            self.Adev = D.CloverField(mem.put(cbuf), X, prec, cmeta, dynamic=True)
            self.A = PR.decode_clover(cbuf, X, prec, cmeta)
            if not dynamic:
                ibuf, imeta = F.clover_to_native(oracle.clover_invert(np.ascontiguousarray(host)), X, prec, compressed=False)
                self.Ainv_dev = D.CloverField(mem.put(ibuf), X, prec, imeta, dynamic=False)
                self.Ainv = PR.decode_clover(ibuf, X, prec, imeta)

    def inv_field(self):
        """(device field, decoded field) that A^-1 is taken from"""
        return (self.Adev, self.A) if self.dynamic else (self.Ainv_dev, self.Ainv)

    def spinor(self, host):
        """oracle-order host spinor (one parity) -> (native field, decoded native-basis value the kernel reads)"""
        buf = F.spinor_to_native(host, self.prec)
        return D.ColorSpinorField(self.mem.put(buf), self.X, self.prec, 1), PR.decode_spinor(buf, self.Vh, self.prec)[0]

    def empty(self):
        return D.ColorSpinorField(self.mem.empty(F.spinor_bytes(self.X, self.prec)), self.X, self.prec, 1)

    def read(self, field, with_norm=False):
        self.mem.sync()
        v, n = PR.decode_spinor(self.mem.get(field.buf), self.Vh, self.prec)
        return (v, n) if with_norm else v


def spinor_kind(X, kind, seed, prec):
    """'gauss' | 'spread' (site magnitudes 2^[-k, k]) | 'points' (a few nonzero sites, exact zeros elsewhere)"""
    if kind == "gauss":
        return PR.gaussian_spinor(X, seed)
    if kind == "spread":
        return PR.gaussian_spinor(X, seed, spread=200 if prec == 8 else 30)
    Vh = F.volume_cb(X)
    return PR.gaussian_spinor(X, seed, points=sorted({0, Vh // 3, Vh - 1, (7 * Vh) // 11}))


def apply_op(Fs, op, be, parity, dagger, din, xd=None, a=0.0, halo=None, mu=0.1, kappa=0.12195, **kw):
    out = Fs.empty()
    if op == "wilson":
        D.ApplyWilson(out, din, Fs.U, a, xd, parity, dagger, halo=halo, backend=be, **kw)
    elif op == "clover":
        D.ApplyWilsonClover(out, din, Fs.U, Fs.Adev, a, xd, parity, dagger, halo=halo, backend=be, **kw)
    elif op == "clover_pc":
        D.ApplyWilsonCloverPreconditioned(out, din, Fs.U, Fs.inv_field()[0], a, xd, parity, dagger, halo=halo, backend=be,
                                          **kw)
    elif op == "tm":
        D.ApplyTwistedMass(out, din, Fs.U, a, 2 * kappa * mu, xd, parity, dagger, halo=halo, backend=be, **kw)
    return out


def reference(Fs, op, parity, dagger, psi, x=None, a=0.0, ghosts=None, mu=0.1, kappa=0.12195):
    p = Fs.prec
    if op == "wilson":
        return PR.wilson(Fs.G, psi, Fs.X, parity, dagger, p, a, x, ghosts)
    if op == "clover":
        return PR.wilson_clover(Fs.G, Fs.A, psi, Fs.X, parity, dagger, p, a, x, ghosts)
    if op == "clover_pc":
        return PR.clover_pc(Fs.G, Fs.inv_field()[1], psi, Fs.X, parity, dagger, p, Fs.dynamic, a, x, ghosts)
    if op == "tm":
        return PR.twisted_mass(Fs.G, psi, Fs.X, parity, dagger, p, a, 2 * kappa * mu, x)
    raise ValueError(op)


def check_op(Fs, op, be, parity=0, dagger=0, kind="gauss", xpay=False, seed=5, what="", mu=0.1, **kw):
    """one application of `op` on a generated spinor; returns max err / bound (asserts <= 1)"""
    psi_h = spinor_kind(Fs.X, kind, seed, Fs.prec)
    din, psi = Fs.spinor(psi_h)
    xd = x = None
    a = 0.0
    if xpay or op in ("clover", "tm"):
        xd, x = Fs.spinor(spinor_kind(Fs.X, kind, seed + 1, Fs.prec))
        a = -0.12195
    out = apply_op(Fs, op, be, parity, dagger, din, xd, a, mu=mu, **kw)
    res = reference(Fs, op, parity, dagger, psi, x, a, mu=mu)
    return PR.assert_within(Fs.read(out), res, Fs.prec, what or f"{op} p={parity} dag={dagger} {kind}")


def check_partitioned(Fs, op, be, comm_dim, split=None, parity=0, dagger=1, seed=31, what=""):
    """self-partitioned run: each decoded ghost face against the projection of the input, then the operator (interior
    + boundary, or the split given) against the reference that reads the decoded ghosts across partitioned faces"""
    psi_h = PR.gaussian_spinor(Fs.X, seed)
    din, psi = Fs.spinor(psi_h)
    xd, x = Fs.spinor(PR.gaussian_spinor(Fs.X, seed + 1))
    a = -0.12195
    halo = ops.self_halo(Fs, Fs.mem, comm_dim)
    ops.self_exchange(Fs, halo, din, 1 - parity, dagger, be)
    Fs.mem.sync()
    ghosts = [[None, None] for _ in range(4)]
    worst = 0.0
    for d in range(4):
        if not comm_dim[d]:
            continue
        face_cb = Fs.Vh * 2 // Fs.X[d] // 2
        for f in range(2):
            h, _ = PR.decode_ghost(Fs.mem.get(halo.ghost[d][f]), face_cb, Fs.prec)
            ghosts[d][f] = h
            ref, T = PR.project_face(psi, Fs.X, 1 - parity, d, 0 if f == 1 else 1, dagger, Fs.prec)
            worst = max(worst, PR.assert_within(h, PR.Result(ref, PR.U_P[Fs.prec] * T), Fs.prec,
                                                f"ghost d={d} f={f}"))
    kws = {"tiles": [dict(kernel=4), dict(kernel=3)], "sites": [dict(kernel=6), dict(kernel=5)],
           "reference": [dict(kernel=1), dict(kernel=2)]}.get(split, [dict()])
    out = Fs.empty()
    for kw in kws:
        if op == "wilson":
            D.ApplyWilson(out, din, Fs.U, a, xd, parity, dagger, halo=halo, backend=be, **kw)
        elif op == "clover_pc":
            D.ApplyWilsonCloverPreconditioned(out, din, Fs.U, Fs.inv_field()[0], a, xd, parity, dagger, halo=halo,
                                              backend=be, **kw)
        else:
            D.ApplyWilsonClover(out, din, Fs.U, Fs.Adev, a, xd, parity, dagger, halo=halo, backend=be, **kw)
    res = reference(Fs, op, parity, dagger, psi, x, a, ghosts)
    if split == "reference" and Fs.prec == 2 and op == "wilson":
        # the interior kernel stores the partial sum x + a D_interior in the half output and the exterior kernel reads
        # it back: one more block-float rounding, of a site whose magnitude is at most |x| + |a| T
        _, T, _ = PR.dslash(Fs.G, psi, Fs.X, parity, dagger, Fs.prec, ghosts)
        mid = PR.Result(np.zeros_like(x), np.abs(x) + abs(a) * T)
        res.bound = res.bound + PR.out_bound(mid, Fs.prec) - mid.bound
    worst = max(worst, PR.assert_within(Fs.read(out), res, Fs.prec, what or f"partitioned {comm_dim} {split} {op}"))
    return worst


def check_multi(Fs, op, be, n_src, parity=1, dagger=0, xpay=True, seed=50, **kw):
    ins, psis, xs, xv = [], [], [], []
    for i in range(n_src):
        d, p = Fs.spinor(PR.gaussian_spinor(Fs.X, seed + i, spread=8))
        ins.append(d)
        psis.append(p)
        d, p = Fs.spinor(PR.gaussian_spinor(Fs.X, seed + 100 + i))
        xs.append(d)
        xv.append(p)
    a = -0.12195 if xpay or op == "clover" else 0.0
    outs = [Fs.empty() for _ in range(n_src)]
    xl = xs if (xpay or op == "clover") else None
    if op == "wilson":
        D.ApplyWilson(outs, ins, Fs.U, a, xl, parity, dagger, backend=be, **kw)
    elif op == "clover_pc":
        D.ApplyWilsonCloverPreconditioned(outs, ins, Fs.U, Fs.inv_field()[0], a, xl, parity, dagger, backend=be, **kw)
    else:
        D.ApplyWilsonClover(outs, ins, Fs.U, Fs.Adev, a, xl, parity, dagger, backend=be, **kw)
    worst = 0.0
    for i in range(n_src):
        res = reference(Fs, op, parity, dagger, psis[i], xv[i] if xl else None, a)
        worst = max(worst, PR.assert_within(Fs.read(outs[i]), res, Fs.prec, f"multi-RHS {op} source {i}/{n_src}"))
    return worst


def check_clover_apply(Fs, be, inverse, parity=1, seed=21, kind="gauss"):
    din, psi = Fs.spinor(spinor_kind(Fs.X, kind, seed, Fs.prec))
    out = Fs.empty()
    if inverse:
        dev, dec = Fs.inv_field()
        D.ApplyClover(out, din, dev, True, parity, backend=be)
        res = PR.clover_apply(dec, psi, parity, True, Fs.dynamic, Fs.prec)
    else:
        D.ApplyClover(out, din, Fs.Adev, False, parity, backend=be)
        res = PR.clover_apply(Fs.A, psi, parity, False, True, Fs.prec)
    return PR.assert_within(Fs.read(out), res, Fs.prec, f"ApplyClover inverse={inverse} {kind}")


def check_twist_gamma(Fs, be, dagger, inverse, kappa=0.12195, mu=0.1, seed=41, kind="gauss"):
    din, psi = Fs.spinor(spinor_kind(Fs.X, kind, seed, Fs.prec))
    out = Fs.empty()
    D.ApplyTwistGamma(out, din, kappa, mu, dagger, inverse, backend=be)
    a, b = PR.twist_coefficients(kappa, mu, dagger, inverse)
    res = PR.twist(psi, a, b, Fs.prec)
    return PR.assert_within(Fs.read(out), res, Fs.prec, f"ApplyTwistGamma mu={mu} dag={dagger} inv={inverse}")
