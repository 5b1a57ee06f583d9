"""The gauge half of an HMC step on one GPU: computeGaugeForceQuda, updateGaugeFieldQuda, momActionQuda and plaqQuda
(lib/interface_quda.cpp) on device tensors; and the measurement that follows a trajectory: the Wilson and Symanzik
gradient flow with the clover energy density and topological charge along it (performWFlowQuda, gaugeObservablesQuda);
and APE, stout, over-improved stout and HYP smearing (performGaugeSmearQuda).

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


# ------------------------------------------------------------------ gradient flow
def _enc(step):
    """signed step +-(d + 1) -> the path code: d forward, 7 - d backward"""
    return step - 1 if step > 0 else 7 + step + 1


def _loops_to_paths(loops):
    return [[_enc(s) for s in loop[1:]] for loop in loops]


def _plaquettes(mu):
    return [[mu + 1, s * (nu + 1), -(mu + 1), -s * (nu + 1)] for nu in range(4) if nu != mu for s in (1, -1)]


def _rectangles(mu):
    out = []
    for nu in range(4):
        if nu == mu:
            continue
        for s in (1, -1):
            m, n = mu + 1, s * (nu + 1)
            out += [[m, m, n, -m, -m, -n], [m, n, -m, -m, -n, m], [m, n, n, -m, -n, -n]]  # each 2x1 loop through the link once
    return out


def _action(kinds):
    paths = [sum((_loops_to_paths(k(mu)) for k, _ in kinds), []) for mu in range(4)]
    coeffs = sum(([c] * len(k(0)) for k, c in kinds), [])
    return paths, coeffs


# name -> (paths[mu][i], coeffs) of the flow action sum_i c_i sum_loops Re tr(1 - loop_i): Wilson (the plaquette, c = 1)
# and Symanzik / Luscher-Weisz (plaquette 5/3, rectangle -1/12), as in the reference's gauge_wilson_flow.cuh
FLOW_ACTIONS = {"wilson": _action([(_plaquettes, 1.0)]),
                "symanzik": _action([(_plaquettes, 5.0 / 3), (_rectangles, -1.0 / 12)])}


def gauge_observables(gauge, *, X, density=None, stream=None, backend=None):
    """gaugeObservablesQuda: {"plaquette": (total, spatial, temporal), "energy": (total, spatial, temporal), "qcharge": Q}.
    energy is the clover E = -sum_planes Re tr(F^2) / V (F = (Q - Q^+) / 8 without its trace, spatial: the planes of two
    spatial directions), Q = sum_x q(x) with q = -1/(4 pi^2) Re (tr F10 F32 - tr F20 F31 + tr F21 F30).  density, a float64
    CUDA tensor of V elements, receives q(x) in parity-major site order."""
    V = int(np.prod(_lattice(X)))
    prec = _check_field("gauge", gauge, (4, V, 3, 3, 2))
    dptr = None
    if density is not None:
        import torch
        if (not isinstance(density, torch.Tensor) or not density.is_cuda or density.dtype != torch.float64
                or density.numel() != V or not density.is_contiguous()):
            raise L.B200Error(f"gauge_observables: density must be a contiguous float64 CUDA tensor of {V} elements")
        dptr = density.data_ptr()
    prefix, lib = backend or ("b200", L.load())
    e, q = (C.c_double * 3)(), C.c_double()
    L.check(getattr(lib, prefix + "_gauge_observables")(e, C.byref(q), dptr, _links(gauge), _lattice(X), prec, stream),
            lib, prefix)
    return {"plaquette": plaquette(gauge, X=X, stream=stream, backend=backend), "energy": tuple(e), "qcharge": q.value}


def gauge_flow(out, gauge, epsilon, n_steps, paths, coeffs, *, X, stream=None, backend=None):
    """n_steps RK3 steps of size epsilon of the gradient flow of the action sum_i coeffs[i] sum_loops Re tr(1 - loop_i),
    the loops given as gauge_force paths, from gauge into out (out may be gauge)"""
    V = int(np.prod(_lattice(X)))
    prec = _check_field("gauge", gauge, (4, V, 3, 3, 2))
    if _check_field("out", out, (4, V, 3, 3, 2)) != prec:
        raise L.B200Error("gauge_flow: out must have the precision of gauge")
    table, lengths, n, max_length = path_table(paths)
    if len(coeffs) != n:
        raise L.B200Error(f"gauge_flow: {n} paths and {len(coeffs)} coefficients")
    prefix, lib = backend or ("b200", L.load())
    L.check(getattr(lib, prefix + "_gauge_flow")(
        _links(out), _links(gauge), _lattice(X), prec, table.ctypes.data_as(C.POINTER(C.c_int)), (C.c_int * n)(*lengths),
        (C.c_double * n)(*[float(c) for c in coeffs]), n, max_length, float(epsilon), int(n_steps), stream), lib, prefix)
    return out


def gradient_flow(gauge, epsilon, n_steps, *, X, action="wilson", meas_interval=0, out=None, stream=None, backend=None):
    """performWFlowQuda: flow gauge by n_steps RK3 steps of size epsilon (Luscher, arXiv:1006.4518) under the action
    FLOW_ACTIONS[action].  Returns (flowed, rows); with meas_interval > 0 a row (t, plaquette, energy, qcharge) of
    gauge_observables is taken at t = 0 and after every meas_interval steps.  out defaults to a new tensor; out=gauge flows
    in place."""
    import torch
    if action not in FLOW_ACTIONS:
        raise L.B200Error(f"gradient_flow: action {action!r} not in {sorted(FLOW_ACTIONS)}")
    n_steps, meas_interval = int(n_steps), int(meas_interval)
    if n_steps < 1 or meas_interval < 0:
        raise L.B200Error("gradient_flow: n_steps must be positive and meas_interval non-negative")
    paths, coeffs = FLOW_ACTIONS[action]
    rows = []

    def measure(g, step):
        o = gauge_observables(g, X=X, stream=stream, backend=backend)
        rows.append((step * float(epsilon), o["plaquette"], o["energy"], o["qcharge"]))

    if meas_interval:
        measure(gauge, 0)
    if out is None:
        out = torch.empty_like(gauge)
    chunk = meas_interval or n_steps
    src, done = gauge, 0
    while done < n_steps:
        k = min(chunk, n_steps - done)
        gauge_flow(out, src, epsilon, k, paths, coeffs, X=X, stream=stream, backend=backend)
        src, done = out, done + k
        if meas_interval and k == meas_interval:
            measure(out, done)
    return out, rows


# ------------------------------------------------------------------ smearing
# kind -> (B200_SMEAR_* code, the coefficient names of its coeff array, dir_ignore when none is given: performGaugeSmearQuda
# smears APE and stout in 3-d with t ignored, over-improved stout and HYP in 4-d)
SMEAR_KINDS = {"ape": (L.SMEAR_APE, ("alpha",), 3), "stout": (L.SMEAR_STOUT, ("rho",), 3),
               "ovrimp_stout": (L.SMEAR_OVRIMP_STOUT, ("rho", "epsilon"), -1),
               "hyp": (L.SMEAR_HYP, ("alpha1", "alpha2", "alpha3"), -1)}


def _smear_kind(kind, dir_ignore):
    if kind not in SMEAR_KINDS:
        raise L.B200Error(f"smearing kind {kind!r} not in {sorted(SMEAR_KINDS)}")
    code, names, default = SMEAR_KINDS[kind]
    if dir_ignore is None or (int(dir_ignore) < 0 and code in (L.SMEAR_APE, L.SMEAR_STOUT)):
        dir_ignore = default
    return code, names, int(dir_ignore)


def gauge_smear(out, gauge, kind, n_steps, *, X, alpha=0.0, rho=0.0, epsilon=0.0, alpha1=0.0, alpha2=0.0, alpha3=0.0,
                dir_ignore=None, stream=None, backend=None):
    """n_steps steps of smearing `kind` (SMEAR_KINDS) from gauge into out (out may be gauge).  APE takes alpha, stout rho,
    over-improved stout rho and epsilon, HYP alpha1, alpha2, alpha3 (alpha1 unused in 3-d).  dir_ignore in 0..3 smears
    only the other three directions and copies the ignored one; 4 smears all four.  None or a negative value is
    performGaugeSmearQuda's default: t ignored for APE and stout, all four directions for over-improved stout and HYP."""
    code, names, dir_ignore = _smear_kind(kind, dir_ignore)
    V = int(np.prod(_lattice(X)))
    prec = _check_field("gauge", gauge, (4, V, 3, 3, 2))
    if _check_field("out", out, (4, V, 3, 3, 2)) != prec:
        raise L.B200Error("gauge_smear: out must have the precision of gauge")
    given = {"alpha": alpha, "rho": rho, "epsilon": epsilon, "alpha1": alpha1, "alpha2": alpha2, "alpha3": alpha3}
    coeff = (C.c_double * 3)(*[float(given[n]) for n in names])
    prefix, lib = backend or ("b200", L.load())
    L.check(getattr(lib, prefix + "_gauge_smear")(_links(out), _links(gauge), _lattice(X), prec, code, coeff, dir_ignore,
                                                  int(n_steps), stream), lib, prefix)
    return out


def smear(gauge, kind, n_steps, *, X, meas_interval=0, out=None, stream=None, backend=None, **coeffs):
    """performGaugeSmearQuda: smear gauge by n_steps steps of `kind` with the coefficients and dir_ignore of gauge_smear.
    Returns (smeared, rows); with meas_interval > 0 a row (step, plaquette, energy, qcharge) of gauge_observables is taken at
    step 0 and after every meas_interval steps.  out defaults to a new tensor; out=gauge smears in place."""
    import torch
    _smear_kind(kind, coeffs.get("dir_ignore"))
    n_steps, meas_interval = int(n_steps), int(meas_interval)
    if n_steps < 1 or meas_interval < 0:
        raise L.B200Error("smear: n_steps must be positive and meas_interval non-negative")
    rows = []

    def measure(g, step):
        o = gauge_observables(g, X=X, stream=stream, backend=backend)
        rows.append((step, o["plaquette"], o["energy"], o["qcharge"]))

    if meas_interval:
        measure(gauge, 0)
    if out is None:
        out = torch.empty_like(gauge)
    chunk = meas_interval or n_steps
    src, done = gauge, 0
    while done < n_steps:
        k = min(chunk, n_steps - done)
        gauge_smear(out, src, kind, k, X=X, stream=stream, backend=backend, **coeffs)
        src, done = out, done + k
        if meas_interval and k == meas_interval:
            measure(out, done)
    return out, rows
