// Gauge half of an HMC step: the gauge force from a table of closed paths, the link update U <- exp(dt P) U, the momentum
// action and the plaquette.  Site code (B2_HD) shared by the CUDA kernels (inst_gauge.cu) and the host twin, plus the
// argument validation and the entry-point bodies of b200_gauge_force / b200_update_gauge / b200_mom_action /
// b200_plaquette.
//
// Reference behaviour reproduced:
//   tests/host_reference/gauge_force_reference.cpp:310-430  path convention (steps 0..3 forward, 7 - d backward, walked
//                                                           from x + mu-hat), mom <- TA(mom - eb3 U_mu(x) sum_i c_i path_i)
//   include/kernels/gauge_update.cuh:35-70                  U <- exp(dt P) U, P the traceless part of mom (its adjoint with
//                                                           conj_mom); order-8 Horner expansion for exact = 0
//   include/kernels/momentum.cuh:41-50                      MILC momentum action 1/2 sum (Im P_kk)^2 + sum_{i<j} |P_ij|^2 - 4
//   lib/gauge_plaq.cu                                       (total, spatial, temporal) mean of Re tr P_mu,nu / 3
// Differences on purpose: the exact exponential is written from Morningstar & Peardon (hep-lat/0311018), with a
// polynomial sin / cos and a Newton solve for cos(acos(r) / 3) built from fma_rn / mul_rn only, so that the CUDA kernels and
// the host twin produce the same bits; the sums are two-stage in a fixed order (clover_build.h's tree), so repeated calls
// give identical results.
//
// Field orders as clover_force.h: links QDP [4][V][3][3][2] (boundary signs included), mom [V][4][10], parity-major sites.
#pragma once

#include "clover_force.h"

namespace b200
{

  // ------------------------------------------------------------------ requests
  struct GaugeForceRequest {
    void *mom;
    const void *qdp[4];
    int X[4];
    const int *paths; // [4][num_paths][max_length]
    const int *length;
    const double *coeff;
    int num_paths, max_length;
    double eb3;
    void *stream;
  };

  struct GaugeUpdateRequest {
    void *out[4];
    const void *in[4];
    const void *mom;
    int X[4];
    double dt;
    int conj_mom, exact;
    void *stream;
  };

  struct GaugeSumRequest { // b200_mom_action (mom) and b200_plaquette (qdp)
    const void *mom;
    const void *qdp[4];
    int X[4];
    void *stream;
  };

  constexpr int kGaugeThreads = kCloverBuildThreads; // threads per CTA; the sums use clover_build.h's per-CTA tree

  // ------------------------------------------------------------------ validation (shared by the library and the host twin)
  inline int check_links(const char *fn, const void *const qdp[4])
  {
    if (!qdp) return set_error(B200_ERR_INVALID, "%s: null argument", fn);
    for (int d = 0; d < 4; d++)
      if (!qdp[d]) return set_error(B200_ERR_INVALID, "%s: link direction %d is NULL", fn, d);
    return 0;
  }

  // the path table of b200_gauge_force / b200_gauge_flow: sizes within the parameter block, finite coefficients, steps in
  // 0..7, every path closed
  inline int check_gauge_paths(const char *fn, const int *paths, const int *length, const double *coeff, int num_paths,
                               int max_length)
  {
    if (!paths || !length || !coeff) return set_error(B200_ERR_INVALID, "%s: null argument", fn);
    if (num_paths < 1 || num_paths > B200_GAUGE_MAX_PATHS)
      return set_error(B200_ERR_INVALID, "%s: num_paths=%d not in [1, %d]", fn, num_paths, B200_GAUGE_MAX_PATHS);
    if (max_length < 1 || max_length > B200_GAUGE_MAX_LENGTH)
      return set_error(B200_ERR_INVALID, "%s: max_length=%d not in [1, %d]", fn, max_length, B200_GAUGE_MAX_LENGTH);
    for (int i = 0; i < num_paths; i++) {
      if (length[i] < 1 || length[i] > max_length)
        return set_error(B200_ERR_INVALID, "%s: length[%d]=%d not in [1, max_length=%d]", fn, i, length[i], max_length);
      if (!std::isfinite(coeff[i])) return set_error(B200_ERR_INVALID, "%s: coeff[%d] is not finite", fn, i);
    }
    for (int mu = 0; mu < 4; mu++) {
      for (int i = 0; i < num_paths; i++) {
        const int *p = paths + ((size_t)mu * num_paths + i) * max_length;
        int disp[4] = {0, 0, 0, 0};
        disp[mu] = 1; // the path starts at x + mu-hat
        for (int j = 0; j < length[i]; j++) {
          if (p[j] < 0 || p[j] > 7)
            return set_error(B200_ERR_INVALID, "%s: step %d of path %d of direction %d is %d, not in [0, 7]", fn, j, i, mu, p[j]);
          if (p[j] < 4) disp[p[j]]++;
          else disp[7 - p[j]]--;
        }
        if (disp[0] || disp[1] || disp[2] || disp[3])
          return set_error(B200_ERR_INVALID, "%s: path %d of direction %d does not close: it ends at x + (%d,%d,%d,%d)", fn, i, mu,
                           disp[0], disp[1], disp[2], disp[3]);
      }
    }
    return 0;
  }

  inline int check_gauge_force(const void *mom, const void *const qdp[4], const int X[4], int precision, const int *paths,
                               const int *length, const double *coeff, int num_paths, int max_length, double eb3)
  {
    const char *fn = "b200_gauge_force";
    if (!mom) return set_error(B200_ERR_INVALID, "%s: null argument", fn);
    if (int rc = check_links(fn, qdp)) return rc;
    if (int rc = check_clover_lattice(fn, X, precision)) return rc;
    if (int rc = check_gauge_paths(fn, paths, length, coeff, num_paths, max_length)) return rc;
    if (!std::isfinite(eb3)) return set_error(B200_ERR_INVALID, "%s: eb3 is not finite", fn);
    return 0;
  }

  inline int check_update_gauge(void *const out[4], const void *const in[4], const void *mom, const int X[4], int precision,
                                double dt)
  {
    const char *fn = "b200_update_gauge";
    if (!mom || !out) return set_error(B200_ERR_INVALID, "%s: null argument", fn);
    for (int d = 0; d < 4; d++)
      if (!out[d]) return set_error(B200_ERR_INVALID, "%s: output direction %d is NULL", fn, d);
    if (int rc = check_links(fn, in)) return rc;
    if (int rc = check_clover_lattice(fn, X, precision)) return rc;
    if (!std::isfinite(dt)) return set_error(B200_ERR_INVALID, "%s: dt is not finite", fn);
    return 0;
  }

  // ------------------------------------------------------------------ kernel arguments
  // The path table is part of the kernel's parameter block (at most 4 KB), which is what bounds B200_GAUGE_MAX_PATHS and
  // B200_GAUGE_MAX_LENGTH; every thread of a CTA walks the same direction's paths, so the table reads are uniform.
  template <typename T> struct GaugeForceArgs {
    CloverBuildArgs<T> g; // links and lattice (border 0)
    T *mom;
    T eb3;
    int num_paths;
    T coeff[B200_GAUGE_MAX_PATHS];
    signed char length[B200_GAUGE_MAX_PATHS];
    signed char step[4][B200_GAUGE_MAX_PATHS][B200_GAUGE_MAX_LENGTH];
  };
  static_assert(sizeof(GaugeForceArgs<double>) <= 4096, "the gauge force arguments must fit the kernel parameter block");

  template <typename T> void fill_lattice(CloverBuildArgs<T> &g, const void *const qdp[4], const int X[4])
  {
    CloverBuildRequest b {};
    for (int d = 0; d < 4; d++) {
      b.qdp[d] = qdp ? qdp[d] : nullptr;
      b.X[d] = X[d];
    }
    fill_clover_build(g, b);
  }

  template <typename T> void fill_gauge_force(GaugeForceArgs<T> &a, const GaugeForceRequest &rq)
  {
    fill_lattice(a.g, rq.qdp, rq.X);
    a.mom = reinterpret_cast<T *>(rq.mom);
    a.eb3 = (T)rq.eb3;
    a.num_paths = rq.num_paths;
    for (int i = 0; i < B200_GAUGE_MAX_PATHS; i++) {
      a.coeff[i] = i < rq.num_paths ? (T)rq.coeff[i] : (T)0;
      a.length[i] = (signed char)(i < rq.num_paths ? rq.length[i] : 0);
    }
    for (int mu = 0; mu < 4; mu++)
      for (int i = 0; i < B200_GAUGE_MAX_PATHS; i++)
        for (int j = 0; j < B200_GAUGE_MAX_LENGTH; j++)
          a.step[mu][i][j] = (signed char)(i < rq.num_paths && j < rq.length[i]
                                             ? rq.paths[((size_t)mu * rq.num_paths + i) * rq.max_length + j] : 0);
  }

  template <typename T> struct GaugeUpdateArgs {
    T *out[4];
    const T *in[4];
    const T *mom;
    T dt;
    int conj_mom, exact, volume_cb;
  };

  template <typename T> void fill_gauge_update(GaugeUpdateArgs<T> &a, const GaugeUpdateRequest &rq)
  {
    for (int d = 0; d < 4; d++) {
      a.out[d] = reinterpret_cast<T *>(rq.out[d]);
      a.in[d] = reinterpret_cast<const T *>(rq.in[d]);
    }
    a.mom = reinterpret_cast<const T *>(rq.mom);
    a.dt = (T)rq.dt;
    a.conj_mom = rq.conj_mom ? 1 : 0;
    a.exact = rq.exact ? 1 : 0;
    a.volume_cb = rq.X[0] * rq.X[1] * rq.X[2] * rq.X[3] / 2;
  }

  // ------------------------------------------------------------------ kernel 1: gauge force -> mom
  // z[d] += delta with periodic wrap; d is a runtime value, so the coordinates are selected in an unrolled loop (a
  // runtime-indexed array would live in local memory)
  B2_HD void shift_coord(int *z, const int *X, int d, int delta)
  {
#pragma unroll
    for (int k = 0; k < 4; k++) {
      if (k != d) continue;
      const int v = z[k] + delta;
      z[k] = v < 0 ? v + X[k] : (v >= X[k] ? v - X[k] : v);
    }
  }

  template <typename T> B2_HD T *mom_at(T *mom, int volume_cb, int x_cb, int parity, int mu)
  {
    return mom + (((size_t)parity * volume_cb + x_cb) * 4 + mu) * 10;
  }

  // f = eb3 U_mu(x) sum_i c_i path_i(x) at coordinates y: the product the gauge force and the gradient flow (gauge_flow.h)
  // project
  template <typename T> B2_HD void gauge_path_sum(T *f, const GaugeForceArgs<T> &a, const int *y, int mu)
  {
    T s[18];
#pragma unroll
    for (int k = 0; k < 18; k++) s[k] = 0;
#pragma unroll 1
    for (int i = 0; i < a.num_paths; i++) {
      int z[4] = {y[0], y[1], y[2], y[3]};
      shift_coord(z, a.g.X, mu, 1);
      T m[18], u[18], t[18];
      const int len = a.length[i];
#pragma unroll 1
      for (int j = 0; j < len; j++) {
        const int st = a.step[mu][i][j];
        const bool fwd = st < 4;
        const int d = fwd ? st : 7 - st;
        if (!fwd) shift_coord(z, a.g.X, d, -1);
        load_link_ext(u, a.g, d, z, 0, 0, 0, 0);
        if (j == 0) {
          if (fwd) {
#pragma unroll
            for (int k = 0; k < 18; k++) m[k] = u[k];
          } else {
            su3_copy_dag(m, u);
          }
        } else {
          if (fwd) su3_mul_op<false, false>(t, m, u);
          else su3_mul_op<false, true>(t, m, u);
#pragma unroll
          for (int k = 0; k < 18; k++) m[k] = t[k];
        }
        if (fwd) shift_coord(z, a.g.X, d, 1);
      }
      const T c = a.coeff[i];
#pragma unroll
      for (int k = 0; k < 18; k++) s[k] = fma_rn(c, m[k], s[k]);
    }
    T u[18];
    load_link_ext(u, a.g, mu, y, 0, 0, 0, 0);
    su3_mul_op<false, false>(f, u, s);
#pragma unroll
    for (int k = 0; k < 18; k++) f[k] = mul_rn(a.eb3, f[k]);
  }

  template <typename T> B2_HD void gauge_force_site(const GaugeForceArgs<T> &a, int x_cb, int parity, int mu)
  {
    Geom geo;
    geom_init(geo, a.g.X);
    int y[4];
    coords_from_cb(y, geo, x_cb, parity);
    T f[18];
    gauge_path_sum(f, a, y, mu);
    mom_sub_ta(mom_at(a.mom, a.g.volume_cb, x_cb, parity, mu), f);
  }

  // ------------------------------------------------------------------ kernel 2: U <- exp(dt P) U
  // sin and cos of x (|x| well below 1e5) from a Cody-Waite reduction by pi/2 and fdlibm's minimax kernels on
  // [-pi/4, pi/4], in fma_rn / mul_rn only: the device's and the host libm's sin / cos need not round alike
  B2_HD void sincos_rn(double x, double &s, double &c)
  {
    constexpr double two_over_pi = 6.36619772367581382433e-01;
    constexpr double pio2_1 = 1.57079632673412561417e+00;  // first 33 bits of pi/2
    constexpr double pio2_1t = 6.07710050650619224932e-11; // pi/2 - pio2_1
    const double k = std::rint(mul_rn(x, two_over_pi));
    const double r = fma_rn(-k, pio2_1t, fma_rn(-k, pio2_1, x));
    const double z = mul_rn(r, r);
    double ps = fma_rn(z, 1.58969099521155010221e-10, -2.50507602534068634195e-08);
    ps = fma_rn(z, ps, 2.75573137070700676789e-06);
    ps = fma_rn(z, ps, -1.98412698298579493134e-04);
    ps = fma_rn(z, ps, 8.33333333332248946124e-03);
    ps = fma_rn(z, ps, -1.66666666666666324348e-01);
    const double sr = fma_rn(mul_rn(z, r), ps, r);
    double pc = fma_rn(z, -1.13596475577881948265e-11, 2.08757232129817482790e-09);
    pc = fma_rn(z, pc, -2.75573143513906633035e-07);
    pc = fma_rn(z, pc, 2.48015872894767294178e-05);
    pc = fma_rn(z, pc, -1.38888888888741095749e-03);
    pc = fma_rn(z, pc, 4.16666666666666019037e-02);
    const double cr = fma_rn(mul_rn(z, z), pc, fma_rn(-0.5, z, 1.0));
    const int q = (int)((long long)k & 3);
    s = q == 0 ? sr : (q == 1 ? cr : (q == 2 ? -sr : -cr));
    c = q == 0 ? cr : (q == 1 ? -sr : (q == 2 ? -cr : sr));
  }

  B2_HD void cmul_rn(double &re, double &im, double ar, double ai, double br, double bi)
  {
    const double r = fma_rn(ar, br, -mul_rn(ai, bi));
    im = fma_rn(ar, bi, mul_rn(ai, br));
    re = r;
  }

  // exp(iQ) = f0 + f1 Q + f2 Q^2 for a traceless Hermitian Q with c0 = det Q, c1 = tr Q^2 / 2 (Morningstar & Peardon,
  // eqs. 19-34).  f[j] = (re, im).
  constexpr double kExpSeriesC1 = 1e-5; // below: the Taylor series to Q^5 (|Q|^6 / 720 < 1e-17) instead of the closed form
  B2_HD void su3_exp_coeffs(double c0, double c1, double (&f)[3][2])
  {
    if (c1 < kExpSeriesC1) { // Q^3 = c1 Q + c0, Q^4 = c1 Q^2 + c0 Q, Q^5 = c1^2 Q + c0 c1 + c0 Q^2; exact identity at Q = 0
      f[0][0] = 1.0;
      f[0][1] = mul_rn(c0, fma_rn(c1, 1.0 / 120, -1.0 / 6));
      f[1][0] = c0 / 24;
      f[1][1] = fma_rn(c1, fma_rn(c1, 1.0 / 120, -1.0 / 6), 1.0);
      f[2][0] = fma_rn(c1, 1.0 / 24, -0.5);
      f[2][1] = c0 / 120;
      return;
    }
    const bool neg = c0 < 0; // f_j(-c0) = (-1)^j conj f_j(c0)
    const double ac0 = neg ? -c0 : c0;
    const double sq = std::sqrt(c1 / 3);
    double r = ac0 / mul_rn(2 * sq, mul_rn(sq, sq)); // c0 / c0_max = cos(theta), theta in [0, pi/2]
    if (r > 1.0) r = 1.0;
    // cos(theta / 3) in [cos(pi/6), 1]: the root of 4 c^3 - 3 c = r, by Newton from c = 1 (monotone, 5 steps reach 1e-23)
    double c = 1.0;
#pragma unroll
    for (int it = 0; it < 6; it++) {
      const double g = fma_rn(mul_rn(4.0, c), mul_rn(c, c), fma_rn(-3.0, c, -r));
      const double gp = fma_rn(mul_rn(12.0, c), c, -3.0);
      c = c - g / gp;
    }
    const double u = mul_rn(sq, c);
    double w2 = mul_rn(c1, fma_rn(-c, c, 1.0)); // c1 sin^2(theta / 3): w enters only through w^2, cos w and sin w / w
    if (w2 < 0) w2 = 0;
    const double w = std::sqrt(w2), u2 = mul_rn(u, u);
    double sw, cw, s2u, c2u, su, cu;
    sincos_rn(w, sw, cw);
    sincos_rn(2 * u, s2u, c2u);
    sincos_rn(u, su, cu);
    // xi0 = sin w / w; its series where the quotient loses digits (M&P eq. 33)
    const double xi0 = w < 0.05 ? fma_rn(-w2 / 6, fma_rn(-w2 / 20, fma_rn(-w2, 1.0 / 42, 1.0), 1.0), 1.0) : sw / w;
    const double emr = cu, emi = -su; // e^{-iu}
    double h[3][2], tr, ti;
    // h0 = (u^2 - w^2) e^{2iu} + e^{-iu} (8 u^2 cos w + 2 i u (3 u^2 + w^2) xi0)
    cmul_rn(tr, ti, emr, emi, mul_rn(mul_rn(8.0, u2), cw), mul_rn(mul_rn(2 * u, fma_rn(3.0, u2, w2)), xi0));
    h[0][0] = fma_rn(u2 - w2, c2u, tr);
    h[0][1] = fma_rn(u2 - w2, s2u, ti);
    // h1 = 2u e^{2iu} - e^{-iu} (2u cos w - i (3 u^2 - w^2) xi0)
    cmul_rn(tr, ti, emr, emi, mul_rn(2 * u, cw), -mul_rn(fma_rn(3.0, u2, -w2), xi0));
    h[1][0] = fma_rn(2 * u, c2u, -tr);
    h[1][1] = fma_rn(2 * u, s2u, -ti);
    // h2 = e^{2iu} - e^{-iu} (cos w + 3 i u xi0)
    cmul_rn(tr, ti, emr, emi, cw, mul_rn(3 * u, xi0));
    h[2][0] = c2u - tr;
    h[2][1] = s2u - ti;
    const double den = fma_rn(9.0, u2, -w2); // >= 2 c1 for theta in [0, pi/2]
#pragma unroll
    for (int j = 0; j < 3; j++) {
      const double re = h[j][0] / den, im = h[j][1] / den;
      f[j][0] = neg && (j & 1) ? -re : re;
      f[j][1] = neg && !(j & 1) ? -im : im;
    }
  }

  // P (18 reals, anti-Hermitian, traceless) of a mom link [10], times sign
  template <typename T> B2_HD void mom_traceless(T *p, const T *m, T sign)
  {
    constexpr int od[3][2] = {{0, 1}, {0, 2}, {1, 2}};
    const T tr = (m[6] + m[7] + m[8]) / (T)3;
#pragma unroll
    for (int k = 0; k < 3; k++) {
      p[(k * 4) * 2] = 0;
      p[(k * 4) * 2 + 1] = sign * (m[6 + k] - tr);
    }
#pragma unroll
    for (int n = 0; n < 3; n++) {
      const int ij = (od[n][0] * 3 + od[n][1]) * 2, ji = (od[n][1] * 3 + od[n][0]) * 2;
      p[ij] = sign * m[2 * n];
      p[ij + 1] = sign * m[2 * n + 1];
      p[ji] = -p[ij];
      p[ji + 1] = p[ij + 1];
    }
  }

  // exp(A) for A = dt P anti-Hermitian traceless, as a 3x3 complex matrix e
  template <typename T> B2_HD void su3_exp(T *e, const T *A)
  {
    T q[18], q2[18]; // Q = -i A (Hermitian)
#pragma unroll
    for (int k = 0; k < 9; k++) {
      q[2 * k] = A[2 * k + 1];
      q[2 * k + 1] = -A[2 * k];
    }
    su3_mul_op<false, false>(q2, q, q);
    const T c1 = (q2[0] + q2[8] + q2[16]) * (T)0.5;
    T t3 = 0; // Re tr(Q Q^2)
#pragma unroll
    for (int i = 0; i < 3; i++) {
#pragma unroll
      for (int j = 0; j < 3; j++) {
        t3 = fma_rn(q[(i * 3 + j) * 2], q2[(j * 3 + i) * 2], t3);
        t3 = fma_rn(-q[(i * 3 + j) * 2 + 1], q2[(j * 3 + i) * 2 + 1], t3);
      }
    }
    double f[3][2];
    su3_exp_coeffs((double)(t3 / (T)3), (double)c1, f);
    const T f0r = (T)f[0][0], f0i = (T)f[0][1], f1r = (T)f[1][0], f1i = (T)f[1][1], f2r = (T)f[2][0], f2i = (T)f[2][1];
#pragma unroll
    for (int k = 0; k < 9; k++) {
      T re = fma_rn(f1r, q[2 * k], -mul_rn(f1i, q[2 * k + 1]));
      T im = fma_rn(f1r, q[2 * k + 1], mul_rn(f1i, q[2 * k]));
      re = fma_rn(f2r, q2[2 * k], re);
      re = fma_rn(-f2i, q2[2 * k + 1], re);
      im = fma_rn(f2r, q2[2 * k + 1], im);
      im = fma_rn(f2i, q2[2 * k], im);
      if (k % 4 == 0) { // diagonal
        re = re + f0r;
        im = im + f0i;
      }
      e[2 * k] = re;
      e[2 * k + 1] = im;
    }
  }

  // order of the Taylor expansion of the reference's exact = 0 update
  constexpr int kUpdateOrder = 8;

  template <typename T> B2_HD void load_link_coherent(T *u, const T *field, size_t site)
  {
    using V = std::conditional_t<sizeof(T) == 8, d2, f2>;
    const V *p = reinterpret_cast<const V *>(field + site * 18);
#pragma unroll
    for (int i = 0; i < 9; i++) { // coherent: out may be in
      const V w = ld<Cache::COHERENT>(p + i);
      u[2 * i] = w.x;
      u[2 * i + 1] = w.y;
    }
  }

  template <typename T> B2_HD void gauge_update_site(const GaugeUpdateArgs<T> &a, int x_cb, int parity, int mu)
  {
    const size_t site = (size_t)parity * a.volume_cb + x_cb;
    T u[18], p[18], r[18], t[18];
    load_link_coherent(u, a.in[mu], site);
    const T *m = a.mom + (site * 4 + mu) * 10;
    mom_traceless(p, m, a.conj_mom ? (T)-1 : (T)1); // conj(P) = P^+ = -P
    if (a.exact) {
#pragma unroll
      for (int k = 0; k < 18; k++) p[k] = mul_rn(a.dt, p[k]);
      su3_exp(t, p);
      su3_mul_op<false, false>(r, t, u);
    } else { // r <- U + (dt / k) P r, k = N .. 1, from r = U
#pragma unroll
      for (int k = 0; k < 18; k++) r[k] = u[k];
#pragma unroll 1
      for (int k = kUpdateOrder; k > 0; k--) {
        const T sc = a.dt / (T)k;
        T sp[18];
#pragma unroll
        for (int l = 0; l < 18; l++) {
          sp[l] = mul_rn(sc, p[l]);
          t[l] = u[l];
        }
        su3_mul_op<false, false, true>(t, sp, r);
#pragma unroll
        for (int l = 0; l < 18; l++) r[l] = t[l];
      }
    }
    T *o = a.out[mu] + site * 18;
#pragma unroll
    for (int k = 0; k < 18; k++) o[k] = r[k];
  }

  // ------------------------------------------------------------------ kernels 3 and 4: the summed site values
  // momentum action of the four links of packed site `site`, in double
  template <typename T> B2_HD double mom_action_site(const T *mom, size_t site)
  {
    double s = 0.0;
#pragma unroll
    for (int mu = 0; mu < 4; mu++) {
      const T *m = mom + (site * 4 + mu) * 10;
      double off = 0.0, dg = 0.0;
#pragma unroll
      for (int j = 0; j < 6; j++) off = fma_rn((double)m[j], (double)m[j], off);
#pragma unroll
      for (int j = 6; j < 9; j++) dg = fma_rn((double)m[j], (double)m[j], dg);
      s += fma_rn(0.5, dg, off) - 4.0;
    }
    return s;
  }

  // sum of Re tr of the plaquettes at (x_cb, parity) over the spatial planes (sp) and the temporal planes (tm), in double
  template <typename T> B2_HD void plaquette_site(const CloverBuildArgs<T> &a, int x_cb, int parity, double &sp, double &tm)
  {
    Geom geo;
    geom_init(geo, a.X);
    int y[4];
    coords_from_cb(y, geo, x_cb, parity);
    sp = 0.0;
    tm = 0.0;
#pragma unroll 1
    for (int p = 0; p < 6; p++) { // planes (1,0), (2,0), (2,1), (3,0), (3,1), (3,2): the clover's first leaf at x
      const PlaneMap m = plane_map(p);
      T q[18];
      leaf_product<0>(q, a, y, m.mu, m.nu);
      const double t = (double)q[0] + (double)q[8] + (double)q[16];
      if (m.mu == 3) tm += t;
      else sp += t;
    }
  }

  // the host's last step of b200_mom_action / b200_plaquette, from the per-group device sums
  inline double mom_action_total(const double g[2]) { return g[0] + g[1]; }
  inline void plaquette_total(double plaq[3], const double g[4], const int X[4])
  {
    const double V = (double)X[0] * X[1] * X[2] * X[3];
    plaq[1] = (g[0] + g[1]) / (9.0 * V);
    plaq[2] = (g[2] + g[3]) / (9.0 * V);
    plaq[0] = 0.5 * (plaq[1] + plaq[2]);
  }

  // ------------------------------------------------------------------ entry points (executor E: the CUDA library or the twin)
  template <typename T> int launch_gauge_force(const GaugeForceRequest &rq);           // inst_gauge.cu
  template <typename T> int launch_gauge_update(const GaugeUpdateRequest &rq);         // inst_gauge.cu
  template <typename T> int launch_mom_action(const GaugeSumRequest &rq, double g[2]); // inst_gauge.cu, synchronises
  template <typename T> int launch_plaquette(const GaugeSumRequest &rq, double g[4]);  // inst_gauge.cu, synchronises

  template <class E>
  int gauge_force(void *mom, const void *const qdp[4], const int X[4], int precision, const int *paths, const int *length,
                  const double *coeff, int num_paths, int max_length, double eb3, void *stream)
  {
    if (int rc = check_gauge_force(mom, qdp, X, precision, paths, length, coeff, num_paths, max_length, eb3)) return rc;
    if (int rc = E::require_device()) return rc;
    GaugeForceRequest rq;
    rq.mom = mom;
    for (int d = 0; d < 4; d++) {
      rq.qdp[d] = qdp[d];
      rq.X[d] = X[d];
    }
    rq.paths = paths;
    rq.length = length;
    rq.coeff = coeff;
    rq.num_paths = num_paths;
    rq.max_length = max_length;
    rq.eb3 = eb3;
    rq.stream = stream;
    return precision == B200_DOUBLE ? E::template gauge_force<double>(rq) : E::template gauge_force<float>(rq);
  }

  template <class E>
  int update_gauge(void *const out[4], const void *const in[4], const void *mom, const int X[4], int precision, double dt,
                   int conj_mom, int exact, void *stream)
  {
    if (int rc = check_update_gauge(out, in, mom, X, precision, dt)) return rc;
    if (int rc = E::require_device()) return rc;
    GaugeUpdateRequest rq;
    for (int d = 0; d < 4; d++) {
      rq.out[d] = out[d];
      rq.in[d] = in[d];
      rq.X[d] = X[d];
    }
    rq.mom = mom;
    rq.dt = dt;
    rq.conj_mom = conj_mom;
    rq.exact = exact;
    rq.stream = stream;
    return precision == B200_DOUBLE ? E::template gauge_update<double>(rq) : E::template gauge_update<float>(rq);
  }

  template <class E> int mom_action(double *S, const void *mom, const int X[4], int precision, void *stream)
  {
    const char *fn = "b200_mom_action";
    if (!S || !mom) return set_error(B200_ERR_INVALID, "%s: null argument", fn);
    if (int rc = check_clover_lattice(fn, X, precision)) return rc;
    if (int rc = E::require_device()) return rc;
    GaugeSumRequest rq {};
    rq.mom = mom;
    for (int d = 0; d < 4; d++) rq.X[d] = X[d];
    rq.stream = stream;
    double g[2];
    const int rc = precision == B200_DOUBLE ? E::template mom_action<double>(rq, g) : E::template mom_action<float>(rq, g);
    if (!rc) *S = mom_action_total(g);
    return rc;
  }

  template <class E> int plaquette(double plaq[3], const void *const qdp[4], const int X[4], int precision, void *stream)
  {
    const char *fn = "b200_plaquette";
    if (!plaq) return set_error(B200_ERR_INVALID, "%s: null argument", fn);
    if (int rc = check_links(fn, qdp)) return rc;
    if (int rc = check_clover_lattice(fn, X, precision)) return rc;
    if (int rc = E::require_device()) return rc;
    GaugeSumRequest rq {};
    for (int d = 0; d < 4; d++) {
      rq.qdp[d] = qdp[d];
      rq.X[d] = X[d];
    }
    rq.stream = stream;
    double g[4];
    const int rc = precision == B200_DOUBLE ? E::template plaquette<double>(rq, g) : E::template plaquette<float>(rq, g);
    if (!rc) plaquette_total(plaq, g, X);
    return rc;
  }

} // namespace b200
