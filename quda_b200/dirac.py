"""Thin Python handles on the C++ operator / solver layer (quda_b200/csrc/host/dirac.h): DiracWilson[PC],
DiracClover[PC], DiracTwistedMass[PC] (reference: lib/dirac_wilson.cpp, lib/dirac_clover.cpp, lib/dirac_twisted_mass.cpp),
CG on the normal equations (lib/inv_cg_quda.cpp), BiCGStab on M itself (lib/inv_bicgstab_quda.cpp) and multi-shift CG on
MdagM + sigma_j (lib/inv_multi_cg_quda.cpp), all mixed-precision with reliable updates.  All arithmetic happens in libquda_b200.so; this module only marshals descriptors."""
import ctypes as C
import math

from . import lib as L

MATPC_EVEN_EVEN, MATPC_ODD_ODD, MATPC_EVEN_EVEN_ASYMMETRIC, MATPC_ODD_ODD_ASYMMETRIC = 0, 1, 2, 3
_TYPES = {"wilson": L.DIRAC_WILSON, "wilsonpc": L.DIRAC_WILSONPC, "clover": L.DIRAC_CLOVER, "cloverpc": L.DIRAC_CLOVERPC,
          "twistedmass": L.DIRAC_TWISTED_MASS, "twistedmasspc": L.DIRAC_TWISTED_MASSPC}


class Dirac:
    def __init__(self, kind, U, kappa, clover=None, clover_inv=None, matpc_type=MATPC_EVEN_EVEN, comm=None, stream=None,
                 mu=0.0):
        self.lib = L.load()
        self.kind, self.U, self.clover, self.clover_inv, self.comm = kind, U, clover, clover_inv, comm  # keep fields alive
        self.prec = U.prec
        h = C.c_void_p()
        X = (C.c_int * 4)(*U.X)
        g = U.desc()
        a = clover.desc() if clover is not None else None
        ai = clover_inv.desc() if clover_inv is not None else None
        L.check(self.lib.b200_dirac_create(C.byref(h), _TYPES[kind], U.prec, X, C.byref(g),
                                           C.byref(a) if a is not None else None,
                                           C.byref(ai) if ai is not None else None, float(kappa), int(matpc_type),
                                           C.byref(comm) if comm is not None else None, stream))
        self.h = h
        if kind.startswith("twistedmass"):
            L.check(self.lib.b200_dirac_set_twist(self.h, float(mu)))

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.lib.b200_dirac_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def _apply(self, what, out, in_, parity=0, x=None, k=0.0, dagger=False):
        o, i = out.desc(), in_.desc()
        xd = x.desc() if x is not None else None
        L.check(self.lib.b200_dirac_apply(self.h, what, C.byref(o), C.byref(i), parity,
                                          C.byref(xd) if xd is not None else None, float(k), int(bool(dagger))))

    def M(self, out, in_, dagger=False):
        self._apply(L.APPLY_M, out, in_, dagger=dagger)

    def Mdag(self, out, in_):
        self._apply(L.APPLY_MDAG, out, in_)

    def MdagM(self, out, in_):
        self._apply(L.APPLY_MDAGM, out, in_)

    def Dslash(self, out, in_, parity, dagger=False):
        self._apply(L.APPLY_DSLASH, out, in_, parity, dagger=dagger)

    def DslashXpay(self, out, in_, parity, x, k, dagger=False):
        self._apply(L.APPLY_DSLASH_XPAY, out, in_, parity, x, k, dagger=dagger)

    def prepare(self, x, b):
        sp, so = C.c_int(-1), C.c_int(-1)
        xd, bd = x.desc(), b.desc()
        L.check(self.lib.b200_dirac_prepare(self.h, C.byref(xd), C.byref(bd), C.byref(sp), C.byref(so)))
        return sp.value, so.value

    def reconstruct(self, x, b):
        xd, bd = x.desc(), b.desc()
        L.check(self.lib.b200_dirac_reconstruct(self.h, C.byref(xd), C.byref(bd)))


def _need_precise(name, precise, fields):
    """The C ABI reads the solution and source fields in the precise operator's precision: refuse any other."""
    for what, f in fields:
        if f.prec != precise.prec:
            raise L.B200Error(f"{name}: {what} has precision {f.prec}, the precise operator {precise.prec}")


def _invert(name, precise, sloppy, x, b, tol, maxiter, delta):
    """Run the C ABI solver b200_<name>; returns the filled SolverParam (iter, true_res, secs, gflops, reliable_updates,
    host_syncs)."""
    _need_precise(name, precise, [("x", x), ("b", b)])
    p = L.SolverParam()
    p.tol, p.maxiter, p.delta = tol, maxiter, delta
    xd, bd = x.desc(), b.desc()
    solve = getattr(precise.lib, "b200_" + name)
    L.check(solve(precise.h, sloppy.h if sloppy is not None else None, C.byref(xd), C.byref(bd), C.byref(p)))
    return p


def invert_cg(precise, sloppy, x, b, tol=1e-10, maxiter=10000, delta=0.1):
    """CG on MdagM x = b (lib/inv_cg_quda.cpp)."""
    return _invert("invert_cg", precise, sloppy, x, b, tol, maxiter, delta)


def invert_bicgstab(precise, sloppy, x, b, tol=1e-10, maxiter=10000, delta=0.1):
    """BiCGStab on M x = b with the operator as given (lib/inv_bicgstab_quda.cpp)."""
    return _invert("invert_bicgstab", precise, sloppy, x, b, tol, maxiter, delta)


def invert_multishift_cg(precise, sloppy, xs, b, offsets, tol=1e-10, tol_offset=None, maxiter=10000, delta=0.1):
    """Multi-shift CG: (MdagM + offsets[j]) xs[j] = b for every shift at once (lib/inv_multi_cg_quda.cpp, with the refinement
    of invertMultiShiftQuda).  The operator is taken as given (the Schur complement for the *pc types).  offsets must be
    finite and non-decreasing; tol_offset (default: tol for every shift) gives each shift its own target.  Every xs[j] is
    overwritten.  Returns the filled MultiShiftParam (iter, iter_offset, refine_iter, iter_res_offset, true_res_offset,
    reliable_updates, secs, gflops, host_syncs)."""
    name = "invert_multishift_cg"
    offsets = [float(o) for o in offsets]
    n = len(offsets)
    if not 1 <= n <= L.MAX_SHIFTS:
        raise L.B200Error(f"{name}: {n} offsets, between 1 and {L.MAX_SHIFTS} are supported")
    if not all(math.isfinite(o) for o in offsets) or any(hi < lo for lo, hi in zip(offsets, offsets[1:])):
        raise L.B200Error(f"{name}: the offsets must be finite and non-decreasing, got {offsets}")
    tols = [float(tol)] * n if tol_offset is None else [float(t) for t in tol_offset]
    if len(tols) != n or not all(t > 0 for t in tols):
        raise L.B200Error(f"{name}: tol_offset needs one positive tolerance per offset, got {tols}")
    if len(xs) != n:
        raise L.B200Error(f"{name}: {len(xs)} solution fields for {n} offsets")
    _need_precise(name, precise, [(f"x[{j}]", x) for j, x in enumerate(xs)] + [("b", b)])
    p = L.MultiShiftParam()
    p.n_shift, p.maxiter, p.delta = n, maxiter, delta
    for j in range(n):
        p.offset[j], p.tol_offset[j] = offsets[j], tols[j]
    xd = (L.Spinor * n)(*[x.desc() for x in xs])
    bd = b.desc()
    L.check(precise.lib.b200_invert_multishift_cg(precise.h, sloppy.h if sloppy is not None else None, xd, C.byref(bd),
                                                  C.byref(p)))
    return p
