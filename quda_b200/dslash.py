"""Python mirror of the reference's Dslash entry points (include/dslash_quda.h:83-921) on top of the C ABI.

`ApplyWilson`, `ApplyWilsonClover`, `ApplyWilsonCloverPreconditioned`, `ApplyClover`, `PackGhost` keep the
reference's names and argument meaning (a == 0 -> no xpay; `parity` = destination parity; `comm_override[d] == 0`
switches communications in dimension d off).  Fields are thin descriptors around device memory owned by the
caller (torch tensors are used for allocation only).  Errors raise B200Error -- the equivalent of errorQuda().

`backend` selects which shared object executes the call: the default (None) is libquda_b200.so on the current
CUDA device.  Tests may pass the CPU "host twin" of the site code explicitly; it is never chosen automatically.
"""
import ctypes as C

import numpy as np

from . import fields as F
from . import lib as L

QUDA_INVALID_PARITY = -1


class Backend:
    def __init__(self, cdll, prefix):
        self.lib, self.prefix = cdll, prefix

    def call(self, name, *args):
        rc = getattr(self.lib, f"{self.prefix}_{name}")(*args)
        L.check(rc, self.lib, self.prefix)


_cuda_backend = None


def cuda_backend():
    global _cuda_backend
    if _cuda_backend is None:
        _cuda_backend = Backend(L.load(), "b200")
    return _cuda_backend


def _ptr(buf):
    if buf is None:
        return None
    if hasattr(buf, "data_ptr"):
        return buf.data_ptr()
    return buf.ctypes.data


class ColorSpinorField:
    """Native-order spinor: n_parity blocks of [24/N planes][volume_cb][N] (+ float norms for half)."""

    def __init__(self, buf, X, prec, n_parity=1):
        self.buf, self.X, self.prec, self.n_parity = buf, [int(v) for v in X], prec, n_parity
        self.volume_cb = F.volume_cb(X)
        self.parity_bytes = F.spinor_bytes(X, prec)

    def desc(self):
        return L.Spinor(_ptr(self.buf), None, self.parity_bytes if self.n_parity == 2 else 0, self.volume_cb, self.n_parity)


class GaugeField:
    def __init__(self, buf, X, prec, recon, meta, anisotropy=1.0, t_boundary=1, first_time_slice=True, last_time_slice=True):
        self.buf, self.X, self.prec, self.recon, self.meta = buf, [int(v) for v in X], prec, recon, meta
        self.anisotropy, self.t_boundary = anisotropy, t_boundary
        self.first_time_slice, self.last_time_slice = first_time_slice, last_time_slice

    def desc(self):
        return L.Gauge(_ptr(self.buf), self.meta["parity_stride_bytes"], self.meta["stride"], self.recon,
                       self.anisotropy, self.meta["link_max"], self.t_boundary, int(self.first_time_slice),
                       int(self.last_time_slice))


class CloverField:
    """Native clover (A or, for static inversion, A^{-1}); `dynamic` -> the inverse is applied by Cholesky solve."""

    def __init__(self, buf, X, prec, meta, dynamic=True):
        self.buf, self.X, self.prec, self.meta, self.dynamic = buf, [int(v) for v in X], prec, meta, dynamic

    def desc(self):
        return L.Clover(_ptr(self.buf), self.meta["parity_stride_bytes"], self.meta["compressed"], int(self.dynamic),
                        self.meta["diagonal"], self.meta["max_element"])


class Halo:
    """Ghost buffers of one field exchange: ghost[d][dir] device buffers (both parities if the field is full).
    For a multi-RHS batch every buffer holds one slab per source, `src_stride[d]` bytes apart (PackGhostMulti fills them
    in one launch); `source(s)` is the view of slab s for a single-source call."""

    def __init__(self):
        self.comm_dim = [0, 0, 0, 0]
        self.ghost = [[None, None] for _ in range(4)]
        self.src, self.src_stride = 0, [0, 0, 0, 0]

    def desc(self, comm_override=None):
        h = L.Halo()
        for d in range(4):
            on = self.comm_dim[d] and (comm_override is None or comm_override[d])
            h.comm_dim[d] = 1 if on else 0
            h.src_stride[d] = int(self.src_stride[d])
            for dir_ in range(2):
                base = _ptr(self.ghost[d][dir_]) if on else None
                h.ghost[d][dir_] = base + self.src * int(self.src_stride[d]) if base is not None else None
                h.ghost_norm[d][dir_] = None
        return h

    def source(self, s):
        h = Halo()
        h.comm_dim, h.ghost, h.src, h.src_stride = self.comm_dim, self.ghost, s, self.src_stride
        return h


def _apply(op, out, in_, U, a, x, parity, dagger, comm_override, A=None, halo=None, kernel=L.KERNEL_AUTO, tile=None,
           stream=None, backend=None, b=0.0, asymmetric=False, fused_dst=None, block_counter=None):
    """`fused_dst` ([4][2] send targets as for PackGhost) and `block_counter` (8 zeroed int32 of pack scratch): run
    pack + interior + boundary as ONE launch (b200_dslash_apply_fused) instead of a separate PackGhost call followed by
    the Dslash."""
    be = backend or cuda_backend()
    multi = isinstance(out, (list, tuple))  # the reference's cvector_ref batch: sources sharing U (and A)
    if multi:
        outs, ins = list(out), list(in_)
        xs = list(x) if x is not None else None
        if len(ins) != len(outs) or (xs is not None and len(xs) != len(outs)):
            raise L.B200Error("multi-RHS: out / in / x batches differ in length")
        out, in_, x = outs[0], ins[0], (xs[0] if xs else None)
    args = L.DslashArgs()
    args.abi_version = L.ABI_VERSION
    args.op, args.kernel, args.precision = op, kernel, out.prec
    for d in range(4):
        args.X[d] = U.X[d]
        args.tile[d] = tile[d] if tile else 0
    args.parity = 0 if parity == QUDA_INVALID_PARITY else parity
    args.dagger = int(bool(dagger))
    args.a = float(a)
    args.b, args.asymmetric = float(b), int(bool(asymmetric))
    args.out, args.in_ = out.desc(), in_.desc()
    if x is not None:
        args.x = x.desc()
    args.U = U.desc()
    if A is not None:
        args.A = A.desc()
    args.halo = (halo or Halo()).desc(comm_override)
    args.stream = stream
    if multi:
        n = len(outs)
        o = (L.Spinor * n)(*[f.desc() for f in outs])
        i = (L.Spinor * n)(*[f.desc() for f in ins])
        xa = (L.Spinor * n)(*[f.desc() for f in xs]) if xs else None
        be.call("dslash_apply_multi", C.byref(args), n, o, i, xa)
    elif fused_dst is not None:
        p = L.PackArgs()
        p.abi_version, p.precision = L.ABI_VERSION, in_.prec
        for d in range(4):
            p.X[d] = in_.X[d]
            p.comm_dim[d] = args.halo.comm_dim[d]
            for f in range(2):
                p.dst[d][f] = _ptr(fused_dst[d][f]) if p.comm_dim[d] else None
        p.parity, p.dagger = 1 - args.parity, args.dagger
        p.in_ = in_.desc()
        p.seq = args.halo.seq
        p.block_counter = _ptr(block_counter)
        p.stream = stream
        be.call("dslash_apply_fused", C.byref(args), C.byref(p))
    else:
        be.call("dslash_apply", C.byref(args))


def ApplyWilson(out, in_, U, a, x, parity, dagger, comm_override=None, halo=None, **kw):
    """out = D in (a == 0) or x + a D in.  Reference: lib/dslash_wilson.cu:9-20.
    `out` / `in_` / `x` may be lists of fields (multi-RHS, the reference's cvector_ref form); likewise below."""
    _apply(L.OP_WILSON, out, in_, U, a, x, parity, dagger, comm_override, halo=halo, **kw)


def ApplyWilsonClover(out, in_, U, A, a, x, parity, dagger, comm_override=None, halo=None, **kw):
    """out = A x + a D in.  Reference: lib/dslash_wilson_clover.cu."""
    _apply(L.OP_CLOVER, out, in_, U, a, x, parity, dagger, comm_override, A=A, halo=halo, **kw)


def ApplyWilsonCloverPreconditioned(out, in_, U, A, a, x, parity, dagger, comm_override=None, halo=None, **kw):
    """out = A^-1 D in (a == 0) or x + a A^-1 D in.  Reference: lib/dslash_wilson_clover_preconditioned.cu:13-27."""
    _apply(L.OP_CLOVER_PC, out, in_, U, a, x, parity, dagger, comm_override, A=A, halo=halo, **kw)


def ApplyTwistedMass(out, in_, U, a, b, x, parity, dagger, comm_override=None, halo=None, **kw):
    """out = a D in + (1 + i b gamma5) x (xpay form only; b is negated for dagger).
    Reference: include/dslash_quda.h:363-365, include/kernels/dslash_twisted_mass.cuh:33-70."""
    _apply(L.OP_TWISTED_MASS, out, in_, U, a, x, parity, dagger, comm_override, halo=halo, b=b, **kw)


def ApplyTwistedMassPreconditioned(out, in_, U, a, b, xpay, x, parity, dagger, asymmetric, comm_override=None, halo=None, **kw):
    """out = a (1 + i b gamma5) D in [+ x]; for dagger without `asymmetric`: out = D^dagger a (1 - i b gamma5) in [+ x].
    Reference: include/dslash_quda.h:403-406, include/kernels/dslash_twisted_mass_preconditioned.cuh:121-175."""
    _apply(L.OP_TWISTED_MASS_PC, out, in_, U, a, x if xpay else None, parity, dagger, comm_override, halo=halo, b=b,
           asymmetric=asymmetric, **kw)


def ApplyClover(out, in_, A, inverse, parity, stream=None, backend=None):
    """out = A in or A^-1 in on one parity.  Reference: lib/dslash_clover_helper.cu:46-54."""
    be = backend or cuda_backend()
    o, i, c = out.desc(), in_.desc(), A.desc()
    be.call("clover_apply", C.byref(o), C.byref(i), C.byref(c), out.prec, int(bool(inverse)), parity, stream)


def ApplyTwistGamma(out, in_, kappa, mu, dagger, inverse, stream=None, backend=None):
    """out = a (1 + i b gamma5) in on one parity: the singlet twist (inverse=False) or its inverse.
    Reference: include/dslash_quda.h:883 (d = 4, epsilon = 0), include/kernels/dslash_gamma_helper.cuh:55-62."""
    be = backend or cuda_backend()
    o, i = out.desc(), in_.desc()
    be.call("twist_gamma5", C.byref(o), C.byref(i), out.prec, float(kappa), float(mu), int(bool(dagger)), int(bool(inverse)), stream)


def PackGhost(dst, in_, parity, dagger, comm_dim, stream=None, backend=None):
    """Spin-project the faces of `in_` (sites of `parity`) into dst[d][face] (local or peer ghost buffers).
    Reference: lib/dslash_pack2.cu:55-425."""
    be = backend or cuda_backend()
    a = L.PackArgs()
    a.abi_version, a.precision = L.ABI_VERSION, in_.prec
    for d in range(4):
        a.X[d] = in_.X[d]
        a.comm_dim[d] = 1 if comm_dim[d] else 0
        for f in range(2):
            a.dst[d][f] = _ptr(dst[d][f]) if comm_dim[d] else None
            a.dst_norm[d][f] = None
    a.parity, a.dagger = parity, int(bool(dagger))
    a.in_ = in_.desc()
    a.stream = stream
    be.call("pack_ghost", C.byref(a))


def PackGhostMulti(dst, ins, parity, dagger, comm_dim, dst_stride, stream=None, backend=None):
    """PackGhost for a multi-RHS batch in ONE launch: source s goes to dst[d][face] + s * dst_stride[d] bytes.
    Reference: lib/dslash_pack2.cu:55-403 (the source index rides in the thread grid)."""
    be = backend or cuda_backend()
    a = L.PackArgs()
    a.abi_version, a.precision = L.ABI_VERSION, ins[0].prec
    for d in range(4):
        a.X[d] = ins[0].X[d]
        a.comm_dim[d] = 1 if comm_dim[d] else 0
        for f in range(2):
            a.dst[d][f] = _ptr(dst[d][f]) if comm_dim[d] else None
            a.dst_norm[d][f] = None
    a.parity, a.dagger = parity, int(bool(dagger))
    a.in_ = ins[0].desc()
    a.stream = stream
    srcs = (L.Spinor * len(ins))(*[f.desc() for f in ins])
    stride = (C.c_size_t * 4)(*[int(v) for v in dst_stride])
    be.call("pack_ghost_multi", C.byref(a), len(ins), srcs, stride)


def copy_spinor(native, host_order, to_native, stream=None):
    """Device-side marshaling between the host interface order ([site][4][3][2], DeGrand-Rossi; a torch tensor of
    float32/float64 on the device) and a native ColorSpinorField.  Reference: lib/copy_color_spinor.cu."""
    lib = L.load()
    d = native.desc()
    hp = host_order.element_size()
    L.check(lib.b200_copy_spinor(C.byref(d), native.prec, host_order.data_ptr(), hp, int(bool(to_native)), stream))


def load_gauge(host_gauge, X, prec, recon, anisotropy=1.0, t_boundary=1, ghost_links=None, first_time_slice=True,
               last_time_slice=True, stream=None):
    """loadGaugeQuda's device work: QDP-order gauge ([4][V][3][3][2], fp64/fp32: a host numpy array, or a CUDA tensor such
    as gauge.update_gauge_field returns, used where it lies) -> resident native GaugeField at (`prec`, `recon`) with the pad
    filled (ghost_links[mu]: neighbour's boundary links, None = periodic self).
    Reference: lib/interface_quda.cpp:571-764, lib/copy_gauge*.cu, lib/extract_gauge_ghost*."""
    import torch
    lib = L.load()
    Vh = F.volume_cb(X)
    pad = F.gauge_pad(X)
    stride = Vh + pad
    if isinstance(host_gauge, torch.Tensor):
        if host_gauge.dtype not in (torch.float64, torch.float32):
            raise L.B200Error("load_gauge: the links must be float64 or float32")
        h = host_gauge.to(device="cuda").contiguous()
        link_max = float(h.abs().max())
    else:
        h = torch.from_numpy(np.ascontiguousarray(host_gauge)).cuda()
        link_max = float(np.abs(host_gauge).max())
    itemsize = h.element_size()
    nbytes = 2 * 4 * recon * stride * prec
    buf = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
    meta = dict(stride=stride, parity_stride_bytes=nbytes // 2, link_max=link_max, pad=pad)
    U = GaugeField(buf, X, prec, recon, meta, anisotropy=anisotropy, t_boundary=t_boundary,
                   first_time_slice=first_time_slice, last_time_slice=last_time_slice)
    d = U.desc()
    Xc = (C.c_int * 4)(*[int(v) for v in X])
    qdp = (C.c_void_p * 4)(*[h[mu].data_ptr() for mu in range(4)])
    keep = []
    gl = (C.c_void_p * 4)()
    for mu in range(4):
        if ghost_links is not None and ghost_links[mu] is not None:
            t = torch.from_numpy(np.ascontiguousarray(ghost_links[mu]).astype(np.float64 if itemsize == 8 else np.float32)).cuda()
            keep.append(t)
            gl[mu] = t.data_ptr()
        else:
            gl[mu] = None
    L.check(lib.b200_copy_gauge(C.byref(d), prec, Xc, qdp, gl, itemsize, stream))
    torch.cuda.synchronize()
    return U


def clover_scale(packed, compressed):
    """(diagonal, max_element) of the native field b200_copy_clover makes from a packed clover [V][2][36] (numpy array or
    torch tensor, evaluated where it lives): the compressed format stores the diagonals as deviations from `diagonal`, and
    max_element is twice the largest stored |value| (CloverField::max_element, clover_field_order.h:621-624)."""
    c = packed.reshape(-1, 36)
    diagonal = float((0.25 * (c[:, 0:3] + c[:, 3:6])).mean()) if compressed else 0.0
    half = 0.5 * (c.double() if hasattr(c, "double") else c.astype(np.float64))
    if compressed:
        mx = max(abs(half[:, 0:3] - diagonal).max(), abs(half[:, 6:30]).max())
    else:
        mx = abs(half).max()
    return diagonal, 2.0 * float(mx)


def _resident_clover(packed_dev, X, prec, compressed, dynamic, diagonal, max_element, stream):
    """packed device clover -> native CloverField at `prec` (b200_copy_clover)"""
    import torch
    lib = L.load()
    CB = 28 if compressed else 36
    nbytes = 2 * 2 * CB * F.volume_cb(X) * prec
    buf = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
    meta = dict(parity_stride_bytes=nbytes // 2, diagonal=diagonal, max_element=max_element, compressed=int(compressed))
    A = CloverField(buf, X, prec, meta, dynamic=dynamic)
    d = A.desc()
    Xc = (C.c_int * 4)(*[int(v) for v in X])
    L.check(lib.b200_copy_clover(C.byref(d), prec, Xc, packed_dev.data_ptr(), packed_dev.element_size(), stream))
    torch.cuda.synchronize()
    return A


def load_clover(host_clover, X, prec, compressed=True, dynamic=True, stream=None):
    """loadCloverQuda's device work: packed host clover (numpy [V][2][36]) -> resident native CloverField.
    Reference: lib/interface_quda.cpp:804-923, lib/copy_clover.cu."""
    import torch
    diagonal, max_element = clover_scale(np.asarray(host_clover), compressed)
    h = torch.from_numpy(np.ascontiguousarray(host_clover)).cuda()
    return _resident_clover(h, X, prec, compressed, dynamic, diagonal, max_element, stream)


def _Xc(X):
    return (C.c_int * 4)(*[int(v) for v in X])


def compute_clover(packed, qdp, X, border, precision, coeff, stream=None, backend=None):
    """packed [V][2][36] = A = 1 + coeff sum sigma F (clover-leaf F) from the QDP-order links qdp ([4][V_e][3][3][2], or four
    per-direction buffers) of the lattice X extended by border[d] in {0, 1} sites per side; fp64 (precision 8) or fp32 (4).
    Reference: lib/interface_quda.cpp:4040-4078 (computeFmunu + computeClover)."""
    be = backend or cuda_backend()
    q = (C.c_void_p * 4)(*[_ptr(qdp[mu]) for mu in range(4)])
    be.call("compute_clover", _ptr(packed), q, _Xc(X), _Xc(border), int(precision), float(coeff), stream)


def clover_invert(inv, packed, X, precision, stream=None, backend=None):
    """inv = A^-1 (inv None: none) of a packed clover by Cholesky; returns [tr log A on even sites, on odd sites].
    Synchronises `stream`.  Reference: lib/clover_invert.cu, include/kernels/clover_invert.cuh."""
    be = backend or cuda_backend()
    tl = (C.c_double * 2)()
    be.call("clover_invert_packed", _ptr(inv), tl, _ptr(packed), _Xc(X), int(precision), stream)
    return [tl[0], tl[1]]


def compute_clover_field(gauge, X, prec, kappa, csw, compressed=True, dynamic=True, grid=None, dist=None, anisotropy=1.0,
                         stream=None):
    """loadCloverQuda(compute_clover=1, compute_clover_inverse=!dynamic): the clover term of the QDP-order links `gauge`
    ([4][V][3][3][2] of the local lattice X, numpy or torch, fp64 / fp32) with coeff = kappa * csw, computed on the device
    in fp64 (prec 8) or fp32 (prec 4, 2).  Returns (A, A^-1 or None, trlog) as resident CloverFields at `prec`; the static
    inverse is stored uncompressed.  With `dist` (torch.distributed) the lattice is the block of `grid` (comm.ProcessGrid):
    the links of the partitioned dimensions are extended by a depth-1 halo (comm.extend_gauge) and trlog is all-reduced.
    Reference: lib/interface_quda.cpp:803-900, 4040-4078."""
    import torch
    if anisotropy != 1.0:
        raise L.B200Error("cannot compute anisotropic clover field")
    hp = F.DOUBLE if prec == F.DOUBLE else F.SINGLE
    dt = torch.float64 if hp == F.DOUBLE else torch.float32
    g = torch.as_tensor(gauge).to(device="cuda", dtype=dt).contiguous()
    border = [0, 0, 0, 0]
    if dist is not None:
        from . import comm
        g = comm.extend_gauge(grid, g, X, dist)
        border = grid.comm_dim()
    packed = torch.empty((2 * F.volume_cb(X), 2, 36), dtype=dt, device="cuda")
    compute_clover(packed, g, X, border, hp, kappa * csw, stream)
    packed_inv = None if dynamic else torch.empty_like(packed)
    trlog = clover_invert(packed_inv, packed, X, hp, stream)
    if dist is not None:
        t = torch.tensor(trlog, dtype=torch.float64, device="cuda" if dist.get_backend() == "nccl" else "cpu")
        dist.all_reduce(t)
        trlog = [float(v) for v in t.cpu()]
    A = _resident_clover(packed, X, prec, compressed, dynamic, *clover_scale(packed, compressed), stream)
    Ainv = None
    if not dynamic:
        Ainv = _resident_clover(packed_inv, X, prec, False, False, *clover_scale(packed_inv, False), stream)
    return A, Ainv, trlog


def flops_per_site(op=L.OP_WILSON, xpay=False):
    """Reference flop model: include/dslash.h:475-528, lib/dslash_wilson_clover_preconditioned.hpp:52-57."""
    f = 1320 + (48 if xpay else 0)
    if op != L.OP_WILSON:
        f += 552
    return f


def min_bytes_per_site(prec, recon, xpay=False, clover_bytes=0):
    """Compulsory traffic B_min = 8 G + 2 S (+S xpay) (+C clover), SURVEY.md 8d / BASELINE.md section 2."""
    G = recon * prec
    S = 24 * prec + (4 if prec == F.HALF else 0)
    return 8 * G + 2 * S + (S if xpay else 0) + clover_bytes
