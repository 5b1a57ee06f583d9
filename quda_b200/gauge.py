"""The gauge half of an HMC step on one GPU: computeGaugeForceQuda, updateGaugeFieldQuda, momActionQuda and plaqQuda
(lib/interface_quda.cpp) on device tensors.

Field orders, shared with dslash.compute_clover_field and dirac.compute_clover_force:
  gauge  [4][V][3][3][2] QDP-order links (fp64 or fp32), parity-major sites, fermion boundary sign included -- every closed
         loop crosses the t boundary an even number of times, so one link field serves the whole trajectory
  mom    [V][4][10] per link the (01), (02), (12) complex entries, the three imaginary diagonals and one pad real
Paths follow the reference's convention: paths[mu][i] is a list of steps, 0..3 forward along that direction and 7 - d
backward along d, walked from x + mu-hat back to x."""
import ctypes as C

import numpy as np

from . import fields as F
from . import lib as L


def _check_field(name, t, shape):
    import torch
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype not in (torch.float64, torch.float32):
        raise L.B200Error(f"{name} must be a float64 or float32 CUDA tensor")
    if tuple(t.shape) != tuple(shape) or not t.is_contiguous():
        raise L.B200Error(f"{name} must be a contiguous tensor of shape {list(shape)}, got {list(t.shape)}")
    return F.DOUBLE if t.element_size() == 8 else F.SINGLE


def _lattice(X):
    if X is None or len(X) != 4:
        raise L.B200Error("the lattice extents X = (x, y, z, t) are needed")
    return (C.c_int * 4)(*[int(v) for v in X])


def _links(g):
    return (C.c_void_p * 4)(*[g[mu].data_ptr() for mu in range(4)])


def path_table(paths):
    """(flat int32 [4][n][max_length], lengths, n, max_length) of paths[mu][i]; every direction has the same number of paths
    and path i the same length in every direction"""
    if len(paths) != 4:
        raise L.B200Error(f"gauge_force: paths needs one list per direction, got {len(paths)}")
    n = len(paths[0])
    if n < 1 or any(len(p) != n for p in paths):
        raise L.B200Error("gauge_force: every direction needs the same, non-zero number of paths")
    lengths = [len(p) for p in paths[0]]
    if any([len(q) for q in p] != lengths for p in paths):
        raise L.B200Error("gauge_force: path i must have the same length in every direction")
    max_length = max(lengths)
    table = np.zeros((4, n, max(max_length, 1)), dtype=np.int32)
    for mu in range(4):
        for i, q in enumerate(paths[mu]):
            table[mu, i, :len(q)] = q
    return table, lengths, n, max_length


def gauge_force(mom, gauge, paths, coeffs, eb3, *, X, stream=None, backend=None):
    """computeGaugeForceQuda: mom <- TA(mom - eb3 U_mu(x) sum_i coeffs[i] path_i(x)) for every link.  With the plaquette
    staples (coefficient 1) and eb3 = dt beta / 3 this is the momentum update of the Wilson action
    beta sum_P (1 - Re tr U_P / 3) over dt, the same kind of update as dirac.compute_clover_force.  mom and gauge are device
    tensors of one precision on the lattice X."""
    V = int(np.prod(_lattice(X)))
    prec = _check_field("mom", mom, (V, 4, 10))
    if _check_field("gauge", gauge, (4, V, 3, 3, 2)) != prec:
        raise L.B200Error("gauge_force: mom and gauge must have the same precision")
    table, lengths, n, max_length = path_table(paths)
    if len(coeffs) != n:
        raise L.B200Error(f"gauge_force: {n} paths and {len(coeffs)} coefficients")
    be = backend or ("b200", L.load())
    prefix, lib = be
    L.check(getattr(lib, prefix + "_gauge_force")(
        mom.data_ptr(), _links(gauge), _lattice(X), prec, table.ctypes.data_as(C.POINTER(C.c_int)),
        (C.c_int * n)(*lengths), (C.c_double * n)(*[float(c) for c in coeffs]), n, max_length, float(eb3), stream),
        lib, prefix)


def update_gauge_field(gauge, mom, dt, conj_mom=False, exact=True, out=None, *, X, stream=None, backend=None):
    """updateGaugeFieldQuda: out[mu] = exp(dt P) gauge[mu] for every link, P the traceless part of mom (of its adjoint with
    conj_mom); exact: the closed-form SU(3) exponential, otherwise the reference's order-8 expansion.  out defaults to a new
    tensor; out=gauge updates in place.  Returns out."""
    import torch
    V = int(np.prod(_lattice(X)))
    prec = _check_field("gauge", gauge, (4, V, 3, 3, 2))
    if _check_field("mom", mom, (V, 4, 10)) != prec:
        raise L.B200Error("update_gauge_field: mom and gauge must have the same precision")
    if out is None:
        out = torch.empty_like(gauge)
    elif _check_field("out", out, (4, V, 3, 3, 2)) != prec:
        raise L.B200Error("update_gauge_field: out must have the precision of gauge")
    prefix, lib = backend or ("b200", L.load())
    L.check(getattr(lib, prefix + "_update_gauge")(_links(out), _links(gauge), mom.data_ptr(), _lattice(X), prec,
                                                  float(dt), int(bool(conj_mom)), int(bool(exact)), stream), lib, prefix)
    return out


def mom_action(mom, *, X=None, stream=None, backend=None):
    """momActionQuda: sum over links of 1/2 sum_k (Im P_kk)^2 + sum_{i<j} |P_ij|^2 - 4 (MILC), in double; a Gaussian momentum
    with this action as exponent has <P_ij> ~ N(0, 1/2) per real component off the diagonal and N(0, 1) on it.  The sum
    depends on the volume only; X defaults to a shape of mom's volume."""
    V = mom.shape[0] if X is None else int(np.prod(_lattice(X)))
    if X is None:
        if V % 16:
            raise L.B200Error(f"mom_action: {V} sites is not the volume of a lattice with even extents")
        X = (V // 8, 2, 2, 2)
    prec = _check_field("mom", mom, (V, 4, 10))
    prefix, lib = backend or ("b200", L.load())
    S = C.c_double()
    L.check(getattr(lib, prefix + "_mom_action")(C.byref(S), mom.data_ptr(), _lattice(X), prec, stream), lib, prefix)
    return S.value


def plaquette(gauge, *, X, stream=None, backend=None):
    """plaqQuda: (total, spatial, temporal) means of Re tr U_P / 3, total = (spatial + temporal) / 2"""
    V = int(np.prod(_lattice(X)))
    prec = _check_field("gauge", gauge, (4, V, 3, 3, 2))
    prefix, lib = backend or ("b200", L.load())
    p = (C.c_double * 3)()
    L.check(getattr(lib, prefix + "_plaquette")(p, _links(gauge), _lattice(X), prec, stream), lib, prefix)
    return tuple(p)
