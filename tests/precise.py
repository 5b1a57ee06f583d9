"""High-precision reference of the Dslash engine's operators with a per-element bound on the kernels' rounding error
(test-only, numpy).

The parity tests elsewhere in the suite use the reference's `compareSpinor` metric: every error is divided by the
largest |element| of the whole field and rounded to a decade.  That accepts an fp32 kernel that is wrong by ~1000 ulp
and a half kernel that is off by several LSBs, and it cannot see errors at sites of small magnitude at all.  This
module checks each output element against its own bound instead.

Pipeline
--------
1. **Decoders** turn the native buffers a kernel reads (DESIGN.md section 3) back into complex arrays in oracle site
   order ([x_cb][spin][colour]), kept in the native (UKQCD) spin basis the kernels compute in; `to_degrand_rossi`
   rotates to the oracle's basis.  They decode exactly: fp64 / fp32 values as stored, half values as q * norm,
   fixed-point links as q / 32767 (x link_max for recon-18), clover values as q * max_element / (2 * 32767).
   Recon-12 and recon-8 links are reconstructed from the stored parameters in the reference precision.
2. **Reference operators** (Wilson hop with dagger / xpay / full field / ghost faces, clover A x and A^-1 x, twisted
   mass, twist_gamma5) run on the decoded inputs in float64 for fp32 and half kernels and in long double for fp64
   kernels, so the only difference between kernel and reference is the kernel's own arithmetic and output rounding.
3. **Bound**, for every real component of every output element:

       |got - ref| <= k_op * u_P * T + Q_out + L_recon

   `u_P` is the unit roundoff of the kernel's arithmetic (2^-53 fp64, 2^-24 fp32 and half, which compute in fp32).
   `T` is the operator applied to absolute values (|U|, |P psi|, |A|, |x|): every rounded intermediate of the kernel is
   a partial sum of terms whose magnitudes T adds up, so a chain of n roundings contributes at most
   gamma_n = n u / (1 - n u) ~ n u times T (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., 3.1).
   For a complex product the real part's terms |ur hr| + |ui hi| are <= |u| |h| (Cauchy-Schwarz), so T built from
   complex moduli bounds the real and imaginary parts alike.

Operation counts (roundings along the longest chain any term passes through)
------------------------------------------------------------------------------
* `K_HOP` = 18 for the Dslash sum of 8 hops: spin projection (1 add; the t projector's factor 2 is exact), the
  SU(3) x half-spinor product as a chain of 6 fused multiply-adds per real component (6), the accumulation of the 8
  hops into the output (8; reconstruction only copies / negates), and up to 3 decode roundings of the inputs: the
  fixed-point link scale (q * 1/32767 rounded and the constant 1/32767 itself rounded to fp32, or link_max
  rounded to fp32), the spinor's block-float norm product, and the deferred-scale product of link and spinor scales.
* `K_XPAY` = 2: x + a * y is a multiply and an add (fused or not).
* `K_CLOVER` = 15 for A x: the chiral basis change (1 add), the 6 x 6 Hermitian product as a chain of 12 real
  operations per component (1 multiply + 11 adds), the basis change back (1 add), and the fixed-point decode of the
  clover entries (1).  Compressed diagonals `diagonal +- deviation` add their own error, carried as a per-entry
  bound (`Clover.err`).
* `K_CHOL` = 4 * (3n + 1) * n + 4 = 460 (n = 6) for the dynamic inverse: the computed solution of a Cholesky solve
  satisfies (H + dH) y = r with |dH| <= gamma_{3n+1} |L| |L^H| (Higham thm. 10.4); ||(|L| |L^H|)||_2 <= n ||H||_2
  and complex arithmetic costs at most 4 real roundings per complex operation, so the normwise forward error is
  <= K_CHOL u kappa_2(H) ||y||_2 per chiral block; the 4 covers the reciprocal square roots on the diagonal.  The
  solve runs in double for fp64 and fp32 clover fields (u = 2^-53) and in float for half (2^-24).  Errors already in
  the right-hand side (the hop sum) propagate through |A^-1|.
* `K_TWIST` = 3: s (v_u - b v_l) is a multiply, an add and a multiply.
* `K_RECON12` = 7 for the third row of recon-12, u0 * conj(row0 x row1): each complex product term is rounded twice
  (multiply + fused multiply-add), the difference once, the scale by u0 once, u0 itself is rounded to the kernel's
  precision (1), and for fixed point each factor carries one decode rounding (2).  It is applied to the |.| version
  of the cross product and propagated through the hop as L_recon.
* Recon-8 is not a short linear chain, so L_recon comes from a running error analysis of the kernel's own
  reconstruction (`_unpack8`): each intermediate carries a bound on its error, with additions and products
  propagated to first order plus the product of the bounds, and the documented errors of the special functions:
  `__sincosf` <= 2^-21.4 absolute on [-pi, pi] (CUDA C Programming Guide, intrinsic functions), `rsqrtf` 2 ulp,
  `__frcp_rn` correctly rounded, double `sincospi` / `rsqrt` 2 ulp.  The cancellation sqrt(1/u0^2 - row_sum) with
  an error c on the argument is bounded by min(sqrt(c), c / m) where m is the exact root.

Output rounding `Q_out`: half an ulp of the stored value, u_P |ref|, for fp32 / fp64.  Half stores q = rint(t * 32767
/ mx) with norm = mx / 32767, so the decoded value is off by 0.5 norm from rounding to an integer, plus the relative
error of the scale: `__fdividef` (2 ulp), the product t * (32767 / mx), the norm product and the constant's rounding
(3 u), times |t| <= mx = 32767 norm.

Propagating a per-part bound through a complex matrix multiplies it by sqrt(2) (the complex modulus of the error).
"""
import numpy as np

from quda_b200 import fields as F

U_P = {8: 2.0 ** -53, 4: 2.0 ** -24, 2: 2.0 ** -24}
K_HOP, K_XPAY, K_CLOVER, K_TWIST, K_RECON12 = 18, 2, 15, 3, 7
K_CHOL = 4 * (3 * 6 + 1) * 6 + 4
FDIVIDEF_ULP = 2
SINCOSF_ABS = 2.0 ** -21.4
RSQRTF_REL = 2 * 2.0 ** -23
PI_LD = np.longdouble("3.14159265358979323846264338327950288")
SQ2 = np.sqrt(2.0)


def real_t(prec):
    """the reference's real type for a kernel precision"""
    return np.longdouble if prec == 8 else np.float64


def cplx_t(prec):
    return np.clongdouble if prec == 8 else np.complex128


# ---------------------------------------------------------------------------------------------- spin algebra (UKQCD)
def proj_rec(mu, sign):
    """(Proj [2x4], Rec [4x2]) with Rec @ Proj = 1 + sign * gamma_mu in the UKQCD basis: the kernel projects a spinor
    to the two spin components h = Proj psi, multiplies h by the link and rebuilds the four components exactly."""
    s, i = float(sign), 1j
    if mu == 0:
        return np.array([[1, 0, 0, s * i], [0, 1, s * i, 0]]), np.array([[1, 0], [0, 1], [0, -s * i], [-s * i, 0]])
    if mu == 1:
        return np.array([[1, 0, 0, s], [0, 1, -s, 0]], complex), np.array([[1, 0], [0, 1], [0, -s], [s, 0]], complex)
    if mu == 2:
        return np.array([[1, 0, s * i, 0], [0, 1, 0, -s * i]]), np.array([[1, 0], [0, 1], [-s * i, 0], [0, s * i]])
    if sign > 0:
        return np.array([[2, 0, 0, 0], [0, 2, 0, 0]], complex), np.array([[1, 0], [0, 1], [0, 0], [0, 0]], complex)
    return np.array([[0, 0, 2, 0], [0, 0, 0, 2]], complex), np.array([[0, 0], [0, 0], [1, 0], [0, 1]], complex)


GAMMA5 = np.array([[0, 0, 1, 0], [0, 0, 0, 1], [1, 0, 0, 0], [0, 1, 0, 0]], complex)  # exchanges the spin pairs
TO_REL = np.array([[0, -1, 0, -1], [1, 0, 1, 0], [0, -1, 0, 1], [1, 0, -1, 0]], float)   # UKQCD -> chiral, x sqrt 2
TO_NONREL = np.array([[0, 1, 0, 1], [-1, 0, -1, 0], [0, 1, 0, -1], [-1, 0, 1, 0]], float)  # chiral -> UKQCD, x sqrt 2


def _dr_matrix():
    """native (UKQCD) -> DeGrand-Rossi: out[s] = (K1[s] v[S1[s]] + K2[s] v[S2[s]]) / sqrt 2"""
    K1, K2, S1, S2 = [-1, 1, 1, 1], [-1, 1, -1, -1], [1, 2, 3, 0], [3, 0, 1, 2]
    R = np.zeros((4, 4), np.longdouble)
    for s in range(4):
        R[s, S1[s]] += K1[s]
        R[s, S2[s]] += K2[s]
    return R / np.sqrt(np.longdouble(2))


_TO_DR = _dr_matrix()


def to_degrand_rossi(v):
    """[..., 4, 3] complex, native basis -> DeGrand-Rossi [..., 4, 3, 2] reals (the oracle's order)"""
    w = np.einsum("ab,...bc->...ac", _TO_DR.astype(v.real.dtype), v)
    return np.stack([w.real, w.imag], axis=-1)


def from_degrand_rossi(host, dtype=np.complex128):
    """oracle [..., 4, 3, 2] reals -> native-basis complex [..., 4, 3]"""
    h = np.asarray(host).astype(np.longdouble)
    c = (h[..., 0] + 1j * h[..., 1]).astype(np.clongdouble)
    return np.einsum("ba,...bc->...ac", _TO_DR, c).astype(dtype)  # _TO_DR is orthogonal


# ---------------------------------------------------------------------------------------------- decoders
def _raw(buf):
    return np.frombuffer(np.ascontiguousarray(buf).tobytes(), dtype=np.uint8)


def decode_spinor(buf, Vh, prec):
    """one native parity block -> (psi [Vh, 4, 3] complex in the native basis, norm [Vh] or None)"""
    raw, N = _raw(buf), F.spinor_N(prec)
    if prec == F.HALF:
        q = raw[: Vh * 48].view(np.int16).reshape(3, Vh, N).transpose(1, 0, 2).reshape(Vh, 24)
        norm = raw[Vh * 48: Vh * 52].view(np.float32)
        flat = q.astype(np.float64) * norm.astype(np.float64)[:, None]  # exact: 16 x 24 bits
    else:
        norm = None
        flat = raw[: Vh * 24 * prec].view(F.real_dtype(prec)).reshape(24 // N, Vh, N).transpose(1, 0, 2).reshape(Vh, 24)
    f = flat.astype(real_t(prec)).reshape(Vh, 12, 2)
    return (f[..., 0] + 1j * f[..., 1]).astype(cplx_t(prec)).reshape(Vh, 4, 3), norm


def decode_ghost(buf, face_cb, prec):
    """one face buffer of one parity -> (h [face_cb, 2, 3] complex, norm or None): 12/N_g planes of N_g-vectors
    (N_g = 2 fp64, 4 fp32 and half), half norms after the 12 * face_cb shorts"""
    raw = _raw(buf)
    Ng = 2 if prec == F.DOUBLE else 4
    if prec == F.HALF:
        q = raw[: face_cb * 24].view(np.int16).reshape(12 // Ng, face_cb, Ng).transpose(1, 0, 2).reshape(face_cb, 12)
        norm = raw[face_cb * 24: face_cb * 28].view(np.float32)
        flat = q.astype(np.float64) * norm.astype(np.float64)[:, None]
    else:
        norm = None
        flat = raw[: face_cb * 12 * prec].view(F.real_dtype(prec)).reshape(12 // Ng, face_cb, Ng).transpose(1, 0, 2)
        flat = flat.reshape(face_cb, 12)
    f = flat.astype(real_t(prec)).reshape(face_cb, 6, 2)
    return (f[..., 0] + 1j * f[..., 1]).astype(cplx_t(prec)).reshape(face_cb, 2, 3), norm


class Gauge:
    """decoded links U[parity][dir][x_cb (incl. pad)][row][col] and a bound on the kernel's reconstruction error of
    every element (zero for recon-18)"""

    def __init__(self, U, err):
        self.U, self.err = U, err


def _u0(X, stride, anisotropy, t_boundary, first_ts, last_ts):
    """u0 factor of every stored link [dir][x_cb]: the anisotropy for space, the t boundary on the last local time
    slice (and for the pad's backward links if this rank holds t = 0)"""
    Vh = F.volume_cb(X)
    t_bound_cb = (X[3] - 1) * X[0] * X[1] * X[2] // 2
    u = np.ones((4, stride))
    u[:3] = anisotropy
    u[3, t_bound_cb:Vh] = t_boundary if last_ts else 1
    u[3, Vh:] = t_boundary if first_ts else 1
    return u


def decode_gauge(buf, X, prec, recon, meta, anisotropy=1.0, t_boundary=1, first_ts=True, last_ts=True):
    """native gauge buffer -> Gauge (complex [2][4][stride][3][3])"""
    stride = meta["stride"]
    N = F.gauge_N(prec, recon)
    M = recon // N
    raw = _raw(buf).view(F.store_dtype(prec)).reshape(2, 4, M, stride, N)
    t = raw.transpose(0, 1, 3, 2, 4).reshape(2, 4, stride, recon).astype(real_t(prec))
    if prec == F.HALF:
        t = t / real_t(prec)(32767)
        if recon == 18:
            t = t * real_t(prec)(meta["link_max"])
    u0 = _u0(X, stride, anisotropy, t_boundary, first_ts, last_ts).astype(real_t(prec))[None, :, :]
    u0 = np.broadcast_to(u0, (2, 4, stride))
    uP = U_P[prec]
    if recon == 8:
        with np.errstate(divide="ignore", invalid="ignore"):  # unused all-zero pad entries
            U, err = _unpack8(t, u0, prec)
        return Gauge(U, err)
    c = (t[..., 0::2] + 1j * t[..., 1::2]).astype(cplx_t(prec))
    if recon == 18:
        return Gauge(c.reshape(2, 4, stride, 3, 3), np.zeros(c.shape[:-1] + (3, 3), real_t(prec)))
    a, b = c[..., 0:3], c[..., 3:6]
    cross = np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                      a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], axis=-1)
    aa, ab = np.abs(a), np.abs(b)
    tcross = np.stack([aa[..., 1] * ab[..., 2] + aa[..., 2] * ab[..., 1], aa[..., 2] * ab[..., 0] + aa[..., 0] * ab[..., 2],
                       aa[..., 0] * ab[..., 1] + aa[..., 1] * ab[..., 0]], axis=-1)
    row2 = u0[..., None] * np.conj(cross)
    U = np.stack([a, b, row2], axis=-2)
    err = np.zeros(U.shape, real_t(prec))
    err[..., 2, :] = K_RECON12 * uP * np.abs(u0)[..., None] * tcross
    return Gauge(U, err)


# running error analysis: (value, bound on the kernel's absolute error in it)
def _add(a, b, u, sub=False):
    v = a[0] - b[0] if sub else a[0] + b[0]
    e = a[1] + b[1]
    return v, e + u * (np.abs(v) + e)


def _mul(a, b, u):
    v = a[0] * b[0]
    e = np.abs(a[0]) * b[1] + np.abs(b[0]) * a[1] + a[1] * b[1]
    return v, e + u * (np.abs(v) + e)


def _neg(a):
    return -a[0], a[1]


def _cmul(a, b, u):
    """complex product as the kernel writes it: re = fma(ar, br, -(ai bi)), im = fma(ar, bi, ai br): the separately
    multiplied term is rounded twice"""
    (ar, ai), (br, bi) = a, b
    re = _add(_mul(ar, br, 0), _mul(ai, bi, u), 0, sub=True)
    im = _add(_mul(ar, bi, 0), _mul(ai, br, u), 0)
    re = (re[0], re[1] + u * (np.abs(re[0]) + re[1]))
    im = (im[0], im[1] + u * (np.abs(im[0]) + im[1]))
    return re, im


def _conj(a):
    return a[0], _neg(a[1])


def _sqrt_diff(d, u, rsqrt_rel):
    """m = sqrt(max(d, 0)) as diff * rsqrt(diff) with the cancellation bound min(sqrt(c), c / m)"""
    v, c = d
    m = np.sqrt(np.maximum(v, 0))
    with np.errstate(divide="ignore", invalid="ignore"):
        prop = np.where(m > 0, np.minimum(np.sqrt(c), c / np.where(m > 0, m, 1)), np.sqrt(c))
    return m, prop + (rsqrt_rel + u) * (m + prop)


def _rcp(a, u):
    v = 1 / a[0]
    e = a[1] / (np.abs(a[0]) * (np.abs(a[0]) - a[1]))
    return v, e + u * (np.abs(v) + e)


def _unpack8(t, u0v, prec):
    """recon-8 reconstruction of the kernel (core.h GaugeView::unpack8) in the reference precision, with a running
    bound on the kernel's error.  Stored: [arg(U10)/pi, arg(-U20)/pi, U11, U12, U00]."""
    rt = real_t(prec)
    u = U_P[prec] if prec != F.DOUBLE else 2.0 ** -53
    zero = np.zeros(t.shape[:-1], rt)
    fixed = prec == F.HALF
    inp = [(t[..., k], (2 * u * np.abs(t[..., k])).astype(rt) if fixed else zero) for k in range(8)]
    u0 = (u0v, (u * np.abs(u0v)).astype(rt) if prec != F.DOUBLE else zero)
    if prec == F.DOUBLE:
        sc_abs, rsq_rel, pi_err = 2 * 2.0 ** -53, 2 * 2.0 ** -53, 0.0
    else:
        sc_abs, rsq_rel, pi_err = SINCOSF_ABS, RSQRTF_REL, abs(float(np.float32(np.pi)) - np.pi)

    def sincospi(x):
        ang = PI_LD.astype(rt) * x[0]
        ea = float(np.pi) * x[1] + pi_err * np.abs(x[0]) + u * np.abs(ang)
        return (np.sin(ang), ea + sc_abs), (np.cos(ang), ea + sc_abs)

    def sq(a):
        return _mul(a, a, 0)

    u0_inv = _rcp(u0, u)
    o1, o2, o3 = (inp[2], inp[3]), (inp[4], inp[5]), (inp[6], inp[7])
    sn, cs = sincospi(inp[0])
    o0 = (cs, sn)
    sn, cs = sincospi(inp[1])
    o6 = (cs, sn)

    def sum4(p, q):  # mul + 3 fma: a term sees at most 4 roundings
        terms = [sq(p[0]), sq(p[1]), sq(q[0]), sq(q[1])]
        v = sum(x[0] for x in terms)
        e = sum(x[1] for x in terms)
        return v, e + 4 * u * (np.abs(v) + e)

    row_sum = sum4(o1, o2)
    row_sum_inv = _rcp(row_sum, u)
    uu = _mul(u0_inv, u0_inv, 0)
    diff = _add(uu, row_sum, u, sub=True)
    m00 = _sqrt_diff(diff, u, rsq_rel)
    o0 = (_mul(o0[0], m00, u), _mul(o0[1], m00, u))
    col_sum = sum4(o0, o3)
    diff = _add(uu, col_sum, u, sub=True)
    m20 = _sqrt_diff(diff, u, rsq_rel)
    o6 = (_mul(o6[0], m20, u), _mul(o6[1], m20, u))
    r_inv2 = _mul(u0_inv, row_sum_inv, u)

    def scale(a, s):
        return _mul(a[0], s, u), _mul(a[1], s, u)

    A = scale(_cmul(_conj(o0), o3, u), u0)
    t4 = _cmul(_conj(o6), _conj(o2), u)
    a1 = _cmul(A, o1, u)
    o4 = tuple(_neg(_mul(r_inv2, _add(t4[k], a1[k], u), u)) for k in range(2))
    t5 = _cmul(_conj(o6), _conj(o1), u)
    a2 = _cmul(A, o2, u)
    o5 = tuple(_mul(r_inv2, _add(t5[k], a2[k], u, sub=True), u) for k in range(2))
    A = scale(_cmul(_conj(o0), o6, u), u0)
    t7 = _cmul(_conj(o3), _conj(o2), u)
    a1 = _cmul(A, o1, u)
    o7 = tuple(_mul(r_inv2, _add(t7[k], a1[k], u, sub=True), u) for k in range(2))
    t8 = _cmul(_conj(o3), _conj(o1), u)
    a2 = _cmul(A, o2, u)
    o8 = tuple(_neg(_mul(r_inv2, _add(t8[k], a2[k], u), u)) for k in range(2))
    rows = [[o3, o4, o5], [o0, o1, o2], [tuple(_neg(x) for x in o6), tuple(_neg(x) for x in o7), tuple(_neg(x) for x in o8)]]
    U = np.empty(t.shape[:-1] + (3, 3), cplx_t(prec))
    E = np.empty(t.shape[:-1] + (3, 3), rt)
    for i in range(3):
        for j in range(3):
            re, im = rows[i][j]
            U[..., i, j] = re[0] + 1j * im[0]
            E[..., i, j] = np.maximum(re[1], im[1])
    return U, E


class Clover:
    """decoded clover: per-site 12 x 12 operator A (native basis, [2][Vh][12][12]), its chiral blocks H
    ([2][Vh][2][6][6], the stored values) and a bound on the kernel's decode error of every block entry"""

    def __init__(self, H, err, prec):
        self.H, self.err, self.prec = H, err, prec


def _tri_pairs():
    """(i, j, slot) of the strictly lower entries in the 36-real block: column major after the 6 diagonals"""
    out, k = [], 6
    for j in range(6):
        for i in range(j + 1, 6):
            out.append((i, j, k))
            k += 2
    return out


TRI = _tri_pairs()


def decode_clover(buf, X, prec, meta):
    Vh = F.volume_cb(X)
    CB = 28 if meta["compressed"] else 36
    N = F.spinor_N(prec)
    rt = real_t(prec)
    raw = _raw(buf).view(F.store_dtype(prec)).reshape(2, 2 * CB // N, Vh, N).transpose(0, 2, 1, 3).reshape(2, Vh, 2, CB)
    st = raw.astype(rt)
    u = U_P[prec]
    e = np.zeros(st.shape, rt)
    if prec == F.HALF:
        st = st * rt(meta["max_element"]) / rt(2 * 32767)
        e = 2 * u * np.abs(st)  # q * nrm rounded in fp32, nrm itself rounded to fp32
    if meta["compressed"]:
        diag = rt(meta["diagonal"])
        a = np.zeros((2, Vh, 2, 36), rt)
        ea = np.zeros_like(a)
        a[..., 0:3] = diag + st[..., 0:3]
        a[..., 3:6] = diag - st[..., 0:3]
        ed = e[..., 0:3] + (0 if prec == F.DOUBLE else 2 * u) * (abs(diag) + np.abs(st[..., 0:3]))
        ea[..., 0:3] = ea[..., 3:6] = ed
        a[..., 6:30] = st[..., 4:28]
        ea[..., 6:30] = e[..., 4:28]
        a[..., 30:34], ea[..., 30:34] = -a[..., 6:10], ea[..., 6:10]
        a[..., 34:36], ea[..., 34:36] = -a[..., 16:18], ea[..., 16:18]
    else:
        a, ea = st, e
    H = np.zeros((2, Vh, 2, 6, 6), cplx_t(prec))
    E = np.zeros((2, Vh, 2, 6, 6), rt)
    for i in range(6):
        H[..., i, i] = a[..., i]
        E[..., i, i] = ea[..., i]
    for i, j, k in TRI:
        H[..., i, j] = a[..., k] + 1j * a[..., k + 1]
        H[..., j, i] = a[..., k] - 1j * a[..., k + 1]
        E[..., i, j] = E[..., j, i] = np.maximum(ea[..., k], ea[..., k + 1])
    return Clover(H, E, prec)


# ---------------------------------------------------------------------------------------------- reference operators
class Result:
    """reference value [Vh, 4, 3] and the bound on every real component of the kernel's result"""

    def __init__(self, ref, bound):
        self.ref, self.bound = ref, bound


def cb_neighbours(X, parity):
    c = F.cb_coords(X, parity)
    fwd, bwd = [], []
    for d in range(4):
        y = c.copy()
        y[:, d] = (c[:, d] + 1) % X[d]
        fwd.append(F.cb_index(y, X))
        y = c.copy()
        y[:, d] = (c[:, d] - 1) % X[d]
        bwd.append(F.cb_index(y, X))
    return c, fwd, bwd


def face_index(c, X, d):
    o = [e for e in range(4) if e != d]
    return ((c[..., o[2]] * X[o[1]] + c[..., o[1]]) * X[o[0]] + c[..., o[0]]) >> 1


def _spin(M, v):
    return np.einsum("ab,nbc->nac", M, v)


def dslash(G, psi, X, parity, dagger, prec, ghosts=None):
    """D psi on the output parity: sum over d of U_d(x) P(d, -+) psi(x + d) + U_d(x - d)^H P(d, +-) psi(x - d), with
    P(d, s) = 1 + s gamma_d (no factor 1/2) and the signs flipped for dagger.  `ghosts[d][f]` (decoded face buffers,
    f = 0 from the backward neighbour, 1 from the forward one) replace the hops across partitioned faces; the
    backward link then comes from the pad.  Returns (D psi, T, L): T the |.| operator, L the propagated recon error."""
    Vh = F.volume_cb(X)
    rt = real_t(prec)
    c, fwd, bwd = cb_neighbours(X, parity)
    out = np.zeros((Vh, 4, 3), cplx_t(prec))
    T = np.zeros((Vh, 4, 3), rt)
    L = np.zeros((Vh, 4, 3), rt)
    apsi = np.abs(psi)
    for d in range(4):
        for is_fwd in (True, False):
            sign = (1 if dagger else -1) if is_fwd else (-1 if dagger else 1)
            Pj, Rc = proj_rec(d, sign)
            Pj, Rc = Pj.astype(cplx_t(prec)), Rc.astype(cplx_t(prec))
            aP, aR = np.abs(Pj).astype(rt), np.abs(Rc).astype(rt)
            if is_fwd:
                U, E, n = G.U[parity, d, :Vh].copy(), G.err[parity, d, :Vh].copy(), fwd[d]
            else:
                U, E, n = G.U[1 - parity, d, bwd[d]], G.err[1 - parity, d, bwd[d]], bwd[d]
            h, ah = _spin(Pj, psi[n]), _spin(aP, apsi[n])
            if ghosts is not None and ghosts[d][0] is not None:
                on = np.nonzero(c[:, d] == (X[d] - 1 if is_fwd else 0))[0]
                fi = face_index(c[on], X, d)
                gh = ghosts[d][1 if is_fwd else 0][fi]
                h[on], ah[on] = gh, np.abs(gh)
                if not is_fwd:
                    U[on], E[on] = G.U[1 - parity, d, Vh + fi], G.err[1 - parity, d, Vh + fi]
            sub = "nij,nsj->nsi" if is_fwd else "nji,nsj->nsi"
            r = np.einsum(sub, U if is_fwd else np.conj(U), h)
            ar = np.einsum(sub, np.abs(U), ah)
            er = np.einsum(sub, E, ah)
            out += _spin(Rc, r)
            T += _spin(aR, ar)
            L += _spin(aR, er)
    return out, T, L


def project_face(psi, X, parity, d, face, dagger, prec):
    """what the pack stores for face `face` (0: x[d] = 0, 1: x[d] = X[d] - 1) of a spinor of parity `parity`: the
    projection the receiving hop needs, in face-index order -> (h [face_cb, 2, 3], T)"""
    c = F.cb_coords(X, parity)
    sel = np.nonzero(c[:, d] == (0 if face == 0 else X[d] - 1))[0]
    fi = face_index(c[sel], X, d)
    sign = (1 if dagger else -1) if face == 0 else (-1 if dagger else 1)
    Pj, _ = proj_rec(d, sign)
    h = np.empty((len(sel), 2, 3), cplx_t(prec))
    T = np.empty((len(sel), 2, 3), real_t(prec))
    h[fi] = _spin(Pj.astype(cplx_t(prec)), psi[sel])
    T[fi] = _spin(np.abs(Pj).astype(real_t(prec)), np.abs(psi[sel]))
    return h, T


def _site_matrix(blocks, prec, scale=1.0):
    """12 x 12 native-basis operator TO_NONREL (x) 1 . blockdiag(blocks) . TO_REL (x) 1 per site"""
    n = blocks.shape[0]
    Hbd = np.zeros((n, 12, 12), blocks.dtype)
    Hbd[:, :6, :6], Hbd[:, 6:, 6:] = blocks[:, 0], blocks[:, 1]
    KN = np.kron(TO_NONREL, np.eye(3)).astype(blocks.real.dtype)
    KR = np.kron(TO_REL, np.eye(3)).astype(blocks.real.dtype)
    return blocks.real.dtype.type(scale) * (KN @ Hbd @ KR), KN, Hbd, KR


def hermitian_inverse(H):
    """inverse of Hermitian positive-definite blocks [..., 6, 6] by Cholesky, in the blocks' own precision
    (np.linalg has no long double)"""
    n = H.shape[-1]
    L = np.zeros_like(H)
    for j in range(n):
        d = H[..., j, j].real - np.sum(np.abs(L[..., j, :j]) ** 2, axis=-1)
        L[..., j, j] = np.sqrt(d)
        for i in range(j + 1, n):
            L[..., i, j] = (H[..., i, j] - np.sum(L[..., i, :j] * np.conj(L[..., j, :j]), axis=-1)) / L[..., j, j]
    Linv = np.zeros_like(H)
    for i in range(n):
        Linv[..., i, i] = 1 / L[..., i, i]
        for j in range(i):
            Linv[..., i, j] = -np.sum(L[..., i, j:i] * Linv[..., j:i, j], axis=-1) / L[..., i, i]
    return np.conj(np.swapaxes(Linv, -1, -2)) @ Linv


def condition(H):
    w = np.linalg.eigvalsh(H.astype(np.complex128))
    return w[..., -1] / w[..., 0]


def _flat(v):
    return v.reshape(v.shape[0], 12)


def clover_apply(A, v, parity, inverse, dynamic, prec, err_in=None):
    """A v or A^-1 v with the clover of one parity -> Result.  `err_in`: bound on an error already in v (a hop sum),
    propagated through |A| or |A^-1|.  Static inverses are fields holding A^-1 and go through inverse=False."""
    rt = real_t(prec)
    u = U_P[prec]
    H, EH = A.H[parity], A.err[parity]
    if inverse and dynamic:
        Hi = hermitian_inverse(H)
        M, KN, Hbd, KR = _site_matrix(Hi, prec, 0.25)
    else:
        M, KN, Hbd, KR = _site_matrix(H, prec)
    x = _flat(v)
    ref = np.einsum("nij,nj->ni", M, x)
    aKN, aKR = np.abs(KN).astype(rt), np.abs(KR).astype(rt)
    ax = np.abs(x)
    TM = np.einsum("ij,njk,kl->nil", aKN, np.abs(Hbd).astype(rt), aKR) * (0.25 if inverse and dynamic else 1)
    bound = np.zeros(ref.shape, rt)
    if inverse and dynamic:
        u_chol = 2.0 ** -24 if prec == F.HALF else 2.0 ** -53
        y = np.einsum("njk,nk->nj", Hbd, np.einsum("ij,nj->ni", KR.astype(x.dtype), x))  # chiral-basis solution
        ynorm = np.sqrt(np.stack([np.sum(np.abs(y[:, :6]) ** 2, -1), np.sum(np.abs(y[:, 6:]) ** 2, -1)], -1))
        kap = condition(H).astype(rt)
        bound += (0.25 * SQ2 * K_CHOL * u_chol * np.sum(kap * ynorm, axis=-1))[:, None]
        bound += 2 * u * np.einsum("nij,nj->ni", TM, ax)           # basis changes + rounding the result
    else:
        bound += K_CLOVER * u * np.einsum("nij,nj->ni", TM, ax)
        EM = np.einsum("ij,njk,kl->nil", aKN, _blockdiag(EH), aKR)
        bound += SQ2 * np.einsum("nij,nj->ni", EM, ax)
    if err_in is not None:
        bound += SQ2 * np.einsum("nij,nj->ni", np.abs(M).astype(rt), _flat(err_in))
    return Result(ref.reshape(v.shape), bound.reshape(v.shape))


def _blockdiag(E):
    out = np.zeros((E.shape[0], 12, 12), E.dtype)
    out[:, :6, :6], out[:, 6:, 6:] = E[:, 0], E[:, 1]
    return out


def twist(v, a, b, prec):
    """a (1 + i b gamma5) v -> Result"""
    rt = real_t(prec)
    ref = rt(a) * (v + 1j * rt(b) * _spin(GAMMA5.astype(v.dtype), v))
    T = abs(rt(a)) * (np.abs(v) + abs(rt(b)) * _spin(GAMMA5.real.astype(rt), np.abs(v)))
    return Result(ref, K_TWIST * U_P[prec] * T)


def wilson(G, psi, X, parity, dagger, prec, a=0.0, x=None, ghosts=None):
    """out = D psi (x is None) or x + a D psi"""
    D, T, L = dslash(G, psi, X, parity, dagger, prec, ghosts)
    u = U_P[prec]
    if x is None:
        return Result(D, K_HOP * u * T + L)
    rt = real_t(prec)
    a = rt(a)
    return Result(x + a * D, (K_HOP + K_XPAY) * u * (np.abs(x) + abs(a) * T) + abs(a) * L)


def wilson_clover(G, A, psi, X, parity, dagger, prec, a, x, ghosts=None):
    """out = A x + a D psi"""
    D, T, L = dslash(G, psi, X, parity, dagger, prec, ghosts)
    Ax = clover_apply(A, x, parity, False, True, prec)
    rt, u = real_t(prec), U_P[prec]
    a = rt(a)
    return Result(Ax.ref + a * D, Ax.bound + K_XPAY * u * np.abs(Ax.ref) + abs(a) * ((K_HOP + K_XPAY) * u * T + L))


def clover_pc(G, A, psi, X, parity, dagger, prec, dynamic, a=0.0, x=None, ghosts=None):
    """out = A^-1 D psi (x is None) or x + a A^-1 D psi; `A` holds A (dynamic) or A^-1 (static)"""
    D, T, L = dslash(G, psi, X, parity, dagger, prec, ghosts)
    u = U_P[prec]
    r = clover_apply(A, D, parity, True, dynamic, prec, err_in=K_HOP * u * T + L)
    if x is None:
        return r
    rt = real_t(prec)
    a = rt(a)
    return Result(x + a * r.ref, abs(a) * r.bound + K_XPAY * u * (np.abs(x) + abs(a) * np.abs(r.ref)))


def twisted_mass(G, psi, X, parity, dagger, prec, a, b, x):
    """ApplyTwistedMass: out = a D psi + (1 + i b' gamma5) x, b' = -b for dagger"""
    D, T, L = dslash(G, psi, X, parity, dagger, prec)
    tw = twist(x, 1.0, -b if dagger else b, prec)
    rt, u = real_t(prec), U_P[prec]
    a = rt(a)
    return Result(tw.ref + a * D, tw.bound + K_XPAY * u * np.abs(tw.ref) + abs(a) * ((K_HOP + K_XPAY) * u * T + L))


def twist_coefficients(kappa, mu, dagger, inverse):
    """(a, b) of ApplyTwistGamma's a (1 + i b gamma5)"""
    b = 2.0 * kappa * mu
    a = 1.0
    if inverse:
        b = -b
        a = 1.0 / (1.0 + b * b)
    return a, (-b if dagger else b)


# ---------------------------------------------------------------------------------------------- the check
def out_bound(res, prec, got_norm=None):
    """add the output rounding Q_out to a Result's bound (per element, real parts)"""
    b = res.bound
    if prec == F.HALF:
        mx = np.max(np.maximum(np.abs(res.ref.real), np.abs(res.ref.imag)) + b, axis=(1, 2))
        rel = 32767 * (FDIVIDEF_ULP * 2.0 ** -23 + 3 * 2.0 ** -24)
        return b + ((0.5 + rel) * mx / 32767 * (1 + 2.0 ** -23))[:, None, None]
    return b + U_P[prec] * np.maximum(np.abs(res.ref.real), np.abs(res.ref.imag))


def ratio(got, res, prec):
    """max over the field of |got - ref| / bound, real and imaginary parts separately (0 / 0 counts as 0)"""
    b = out_bound(res, prec)
    d = np.maximum(np.abs((got - res.ref).real), np.abs((got - res.ref).imag)).astype(np.float64)
    b = b.astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(d == 0, 0.0, d / b)
    return float(np.max(r)) if r.size else 0.0


def assert_within(got, res, prec, what):
    r = ratio(got, res, prec)
    print(f"{what}: max err/bound = {r:.3g}")
    assert np.all(np.isfinite(got)), f"{what}: non-finite output"
    assert r <= 1.0, f"{what}: max err/bound = {r:.4g} > 1"
    return r


# ---------------------------------------------------------------------------------------------- field generators
def _rng(seed):
    return np.random.default_rng(seed)


def gaussian_spinor(X, seed, nparity=1, spread=0, points=None):
    """signed Gaussian spinor in oracle order [n][4][3][2]; `spread` k: each site scaled by 2^j, j uniform in [-k, k];
    `points`: list of site indices that stay nonzero (every other site is exactly zero)"""
    r = _rng(seed)
    n = F.volume_cb(X) * nparity
    s = r.standard_normal((n, 4, 3, 2))
    if spread:
        s *= np.exp2(r.integers(-spread, spread + 1, n)).reshape(n, 1, 1, 1)
    if points is not None:
        keep = np.zeros(n, bool)
        keep[list(points)] = True
        s[~keep] = 0.0
    return s


def _su3_haar(n, r):
    z = (r.standard_normal((n, 3, 3)) + 1j * r.standard_normal((n, 3, 3))) / np.sqrt(2)
    q, rr = np.linalg.qr(z)
    d = np.diagonal(rr, axis1=-2, axis2=-1)
    q = q * (d / np.abs(d))[:, None, :]
    det = np.linalg.det(q)
    return q / (det ** (1.0 / 3.0))[:, None, None]


def _su3_near_identity(n, r, eps):
    h = r.standard_normal((n, 3, 3)) + 1j * r.standard_normal((n, 3, 3))
    h = 0.5 * (h + np.conj(np.swapaxes(h, 1, 2)))
    h -= (np.trace(h, axis1=1, axis2=2) / 3)[:, None, None] * np.eye(3)
    w, v = np.linalg.eigh(h)
    return np.einsum("nij,nj,nkj->nik", v, np.exp(1j * eps * w), np.conj(v))


def random_gauge(X, seed, eps=None, anisotropy=1.0, antiperiodic_t=True):
    """QDP-order gauge [4][V][3][3][2]: Haar-random SU(3) (eps None) or exp(i eps H); spatial links / anisotropy and
    the last time slice's t links negated for antiperiodic t (the oracle's conventions)"""
    r = _rng(seed)
    V = 2 * F.volume_cb(X)
    U = _su3_haar(4 * V, r) if eps is None else _su3_near_identity(4 * V, r, eps)
    U = U.reshape(4, V, 3, 3)
    U[:3] /= anisotropy
    if antiperiodic_t:
        for p in range(2):
            c = F.cb_coords(X, p)
            last = np.nonzero(c[:, 3] == X[3] - 1)[0] + p * (V // 2)
            U[3, last] *= -1
    return np.ascontiguousarray(np.stack([U.real, U.imag], axis=-1))


def hpd_clover(X, seed, cond):
    """host-order clover [V][2][36] whose chiral blocks are Q diag Q^H with eigenvalues spread log-uniformly over
    [1, cond] (times 0.5..1): Hermitian positive definite with condition number `cond`"""
    r = _rng(seed)
    V = 2 * F.volume_cb(X)
    Q = _su3_haar_n(2 * V, 6, r)
    lam = np.exp(np.linspace(0, np.log(cond), 6))[None, :] * r.uniform(0.5, 1.0, (2 * V, 1))
    H = np.einsum("nij,nj,nkj->nik", Q, lam, np.conj(Q)).reshape(V, 2, 6, 6)
    out = np.zeros((V, 2, 36))
    for i in range(6):
        out[..., i] = H[..., i, i].real
    for i, j, k in TRI:
        out[..., k], out[..., k + 1] = H[..., i, j].real, H[..., i, j].imag
    return out


def _su3_haar_n(n, dim, r):
    z = (r.standard_normal((n, dim, dim)) + 1j * r.standard_normal((n, dim, dim))) / np.sqrt(2)
    q, rr = np.linalg.qr(z)
    d = np.diagonal(rr, axis1=-2, axis2=-1)
    return q * (d / np.abs(d))[:, None, :]
