// APE, stout, over-improved stout and HYP smearing of a gauge field.  Site code (B2_HD) shared by the CUDA kernels
// (inst_gauge_smear.cu) and the host twin, the argument validation, the launch sequence both executors run, and the
// entry-point body of b200_gauge_smear.
//
// Behaviour reproduced (S_mu(x): the sum of the staples of U_mu(x) in the smeared planes, d = 4, or 3 with dir_ignore):
//   include/kernels/gauge_ape.cuh:51-83        APE: U' = P[(1 - alpha) 1 + alpha / (2 (d - 1)) S U^+] U
//   include/kernels/gauge_stout.cuh:61-93      stout: U' = exp(rho TA(S U^+)) U, i.e. one Euler step of the Wilson flow
//   include/kernels/gauge_stout.cuh:140-177    over-improved stout (Moran & Leinweber, arXiv:0801.1165): the same with
//                                              (rho (5 - 2 eps) / 3) S - (rho (1 - eps) / 12) R, R the 2x1 rectangle staples
//   include/kernels/gauge_hyp.cuh,             HYP (Hasenfratz & Knechtli, hep-lat/0103029), every level
//   lib/gauge_hyp.cu:101-146                   U' = P[(1 - alpha) 1 + c staple U^+] U with U the thin link: 4-d in three
//                                              levels (alpha3 / 2, alpha2 / 4, alpha1 / 6), 3-d in two (alpha3 / 2, alpha2 / 4)
//   include/su3_project.cuh:85-109             P: the unitary polar factor by the Newton iteration W <- (W + W^-+) / 2
//                                              (tolerance 2e-15 in fp64, 1e-6 in fp32, at most 100 iterations), divided by
//                                              the principal cube root of its determinant (arg in (-pi, pi])
// Differences on purpose: the cube root of the determinant is built from fma_rn / mul_rn, division and sqrt only (a Newton
// cos(theta / 3) as in su3_exp_coeffs, no libm transcendental), so the CUDA kernels and the host twin produce the same
// bits; the ignored direction is copied bit for bit.
//
// Projecting the product with U^+ rather than the link sum is what carries the fermion boundary sign: S U^+ is unchanged
// when U and its staples change sign together, whereas det(-A) = -det A would select another centre element.
//
// Field orders as gauge.h: links QDP [4][V][3][3][2] (boundary signs included), parity-major sites.  Decorated HYP links
// are [slot][V][3][3][2], slot(mu, v) numbering the links (mu, v != mu) of the smeared directions.
#pragma once

#include "gauge_flow.h"

namespace b200
{

  // ------------------------------------------------------------------ request
  struct GaugeSmearRequest {
    void *out[4];
    const void *in[4];
    int X[4];
    int type;        // B200_SMEAR_*
    double coeff[3]; // {alpha}, {rho}, {rho, epsilon} or {alpha1, alpha2, alpha3}
    int ign;         // the direction left unsmeared, 4: none
    int n_steps;
    void *stream;
  };

  inline int smear_coeff_count(int type) { return type == B200_SMEAR_HYP ? 3 : (type == B200_SMEAR_OVRIMP_STOUT ? 2 : 1); }

  // ------------------------------------------------------------------ validation (shared by the library and the host twin)
  inline int check_gauge_smear(void *const out[4], const void *const in[4], const int X[4], int precision, int type,
                               const double *coeff, int dir_ignore, int n_steps)
  {
    const char *fn = "b200_gauge_smear";
    if (!out || !coeff) return set_error(B200_ERR_INVALID, "%s: null argument", fn);
    for (int d = 0; d < 4; d++)
      if (!out[d]) return set_error(B200_ERR_INVALID, "%s: output direction %d is NULL", fn, d);
    if (int rc = check_links(fn, in)) return rc;
    if (int rc = check_clover_lattice(fn, X, precision)) return rc;
    if (type < B200_SMEAR_APE || type > B200_SMEAR_HYP) return set_error(B200_ERR_INVALID, "%s: unknown smearing type %d", fn, type);
    for (int i = 0; i < smear_coeff_count(type); i++)
      if (!std::isfinite(coeff[i])) return set_error(B200_ERR_INVALID, "%s: coeff[%d] is not finite", fn, i);
    if (dir_ignore < -1 || dir_ignore > 4) return set_error(B200_ERR_INVALID, "%s: dir_ignore=%d not in [-1, 4]", fn, dir_ignore);
    if (n_steps < 1) return set_error(B200_ERR_INVALID, "%s: n_steps=%d must be at least 1", fn, n_steps);
    return 0;
  }

  // ------------------------------------------------------------------ SU(3) projection
  template <typename T> constexpr T kProjectTol = sizeof(T) == 8 ? (T)2e-15 : (T)1e-6;
  constexpr int kProjectMaxIter = 100;

  // (re, im) of a b - c d for complex a, b, c, d given by their offsets into the 3x3 matrix m
  template <typename T> B2_HD void cdet2(T &re, T &im, const T *m, int a, int b, int c, int d)
  {
    const T pr = fma_rn(m[a], m[b], -mul_rn(m[a + 1], m[b + 1])), pi = fma_rn(m[a], m[b + 1], mul_rn(m[a + 1], m[b]));
    const T qr = fma_rn(m[c], m[d], -mul_rn(m[c + 1], m[d + 1])), qi = fma_rn(m[c], m[d + 1], mul_rn(m[c + 1], m[d]));
    re = pr - qr;
    im = pi - qi;
  }

  // inv = a^-1 by cofactors, and det a
  template <typename T> B2_HD void su3_inverse(T *inv, T &dr, T &di, const T *a)
  {
    T cof[18]; // cof[i][j] = the cofactor of a[j][i]
#pragma unroll
    for (int i = 0; i < 3; i++) {
#pragma unroll
      for (int j = 0; j < 3; j++) {
        const int j1 = (j + 1) % 3, j2 = (j + 2) % 3, i1 = (i + 1) % 3, i2 = (i + 2) % 3;
        cdet2(cof[(i * 3 + j) * 2], cof[(i * 3 + j) * 2 + 1], a, (j1 * 3 + i1) * 2, (j2 * 3 + i2) * 2, (j1 * 3 + i2) * 2,
              (j2 * 3 + i1) * 2);
      }
    }
    dr = 0;
    di = 0;
#pragma unroll
    for (int k = 0; k < 3; k++) { // det = sum_k a[0][k] cof(a[0][k])
      const T ar = a[k * 2], ai = a[k * 2 + 1], cr = cof[(k * 3) * 2], ci = cof[(k * 3) * 2 + 1];
      dr = fma_rn(ar, cr, fma_rn(-ai, ci, dr));
      di = fma_rn(ar, ci, fma_rn(ai, cr, di));
    }
    const T n = fma_rn(dr, dr, mul_rn(di, di));
    const T ir = dr / n, ii = -di / n;
#pragma unroll
    for (int k = 0; k < 9; k++) {
      inv[2 * k] = fma_rn(cof[2 * k], ir, -mul_rn(cof[2 * k + 1], ii));
      inv[2 * k + 1] = fma_rn(cof[2 * k], ii, mul_rn(cof[2 * k + 1], ir));
    }
  }

  // the reference's stopping rule: W = (W^-1)^+ and W^+ W = 1, every component to tol
  template <typename T> B2_HD bool su3_is_unitary(const T *w, const T *inv, T tol)
  {
#pragma unroll
    for (int i = 0; i < 3; i++) {
#pragma unroll
      for (int j = 0; j < 3; j++) {
        const int ij = (i * 3 + j) * 2, ji = (j * 3 + i) * 2;
        if (std::fabs(w[ij] - inv[ji]) > tol || std::fabs(w[ij + 1] + inv[ji + 1]) > tol) return false;
      }
    }
    T p[18];
    su3_mul_op<true, false>(p, w, w);
#pragma unroll
    for (int i = 0; i < 3; i++) {
#pragma unroll
      for (int j = 0; j < 3; j++) {
        const int ij = (i * 3 + j) * 2;
        if (std::fabs(p[ij] - (i == j ? (T)1 : (T)0)) > tol || std::fabs(p[ij + 1]) > tol) return false;
      }
    }
    return true;
  }

  // (cos, sin) of theta / 3 for the unit complex number (c, s) = e^{i theta}, theta in (-pi, pi] (s = -0 counts as +0).
  // With alpha = theta or pi - |theta| in [0, pi/2], cos(alpha / 3) is the root of 4 x^3 - 3 x = cos(alpha) in
  // [cos(pi/6), 1], where Newton from x = 1 converges monotonically (su3_exp_coeffs' solve), and
  // sin(alpha / 3) = sin(alpha) / (4 x^2 - 1) with 4 x^2 - 1 in [2, 3]; theta / 3 = pi/3 - alpha / 3 on the left half-plane.
  B2_HD void third_angle(double c, double s, double &c3, double &s3)
  {
    const bool left = c < 0;
    const double r = left ? -c : c, sa = s < 0 ? -s : s;
    double x = 1.0;
#pragma unroll
    for (int it = 0; it < 6; it++) {
      const double g = fma_rn(mul_rn(4.0, x), mul_rn(x, x), fma_rn(-3.0, x, -r));
      const double gp = fma_rn(mul_rn(12.0, x), x, -3.0);
      x = x - g / gp;
    }
    const double y = sa / fma_rn(mul_rn(4.0, x), x, -1.0);
    constexpr double h = 0.86602540378443864676; // sin(pi/3)
    c3 = left ? fma_rn(0.5, x, mul_rn(h, y)) : x;
    s3 = left ? fma_rn(h, x, mul_rn(-0.5, y)) : y;
    if (s < 0) s3 = -s3;
  }

  // p = the SU(3) projection of w: the unitary polar factor by Newton's iteration, over the principal cube root of its det
  template <typename T> B2_HD void su3_project(T *p, const T *w0, T tol)
  {
    T w[18], inv[18], dr, di;
#pragma unroll
    for (int k = 0; k < 18; k++) w[k] = w0[k];
    su3_inverse(inv, dr, di, w);
#pragma unroll 1
    for (int it = 0; it < kProjectMaxIter; it++) {
#pragma unroll
      for (int i = 0; i < 3; i++) {
#pragma unroll
        for (int j = 0; j < 3; j++) {
          const int ij = (i * 3 + j) * 2, ji = (j * 3 + i) * 2;
          w[ij] = mul_rn((T)0.5, w[ij] + inv[ji]);
          w[ij + 1] = mul_rn((T)0.5, w[ij + 1] - inv[ji + 1]);
        }
      }
      su3_inverse(inv, dr, di, w);
      if (su3_is_unitary(w, inv, tol)) break;
    }
    // det w = m e^{i theta}: multiply by m^{-1/3} e^{-i theta / 3}; m^{-1/3} by Newton on m y^3 = 1 from y = 1 (|m - 1| is of
    // the order of tol)
    const double xr = (double)dr, xi = (double)di;
    const double m = std::sqrt(fma_rn(xr, xr, mul_rn(xi, xi)));
    double c3, s3, y = 1.0;
    third_angle(xr / m, xi / m, c3, s3);
#pragma unroll
    for (int it = 0; it < 5; it++) {
      const double my2 = mul_rn(m, mul_rn(y, y));
      y = y - fma_rn(my2, y, -1.0) / mul_rn(3.0, my2);
    }
    const T zr = (T)mul_rn(y, c3), zi = (T)mul_rn(-y, s3);
#pragma unroll
    for (int k = 0; k < 9; k++) {
      p[2 * k] = fma_rn(zr, w[2 * k], -mul_rn(zi, w[2 * k + 1]));
      p[2 * k + 1] = fma_rn(zr, w[2 * k + 1], mul_rn(zi, w[2 * k]));
    }
  }

  // ------------------------------------------------------------------ kernel 1: stout and over-improved stout
  // out_mu(x) = exp(-TA(rho U_mu(x) sum_i c_i path_i)) U_mu(x), the paths the staples of the smeared planes (and their
  // rectangles): exp(rho TA(S U^+)) U, the Euler step of the flow generator of gauge_flow.h
  template <typename T> struct GaugeStoutArgs {
    GaugeForceArgs<T> f; // this step's input links (f.g), the staple table and rho (f.eb3); f.mom unused
    T *out[4];
    int ign;
  };
  static_assert(sizeof(GaugeStoutArgs<double>) <= 4096, "the stout arguments must fit the kernel parameter block");

  // the direction of grid row y (the smeared directions in order, ign skipped)
  B2_HD int smear_dir(int y, int ign) { return y + (y >= ign ? 1 : 0); }

  // the staple table of one smearing: per direction mu the plaquette staples of the planes (mu, nu), nu != mu, ign, with
  // coefficient cp, then (rect) their 2x1 rectangles with cr, in the order of gauge.py's FLOW_ACTIONS.  The row of the
  // ignored direction is filled like the others and never read.
  struct SmearPaths {
    int n, max_length;
    int length[B200_GAUGE_MAX_PATHS];
    double coeff[B200_GAUGE_MAX_PATHS];
    int steps[4][B200_GAUGE_MAX_PATHS][5];
  };

  inline void smear_paths(SmearPaths &t, int ign, bool rect, double cp, double cr)
  {
    auto enc = [](int s) { return s > 0 ? s - 1 : 7 + s + 1; }; // signed step +-(d + 1) -> d forward, 7 - d backward
    const int nplanes = ign < 4 ? 2 : 3;
    for (int mu = 0; mu < 4; mu++) {
      int n = 0, planes = 0;
      const int m = mu + 1;
      for (int kind = 0; kind < (rect ? 2 : 1); kind++) {
        planes = 0;
        for (int nu = 0; nu < 4 && planes < nplanes; nu++) {
          if (nu == mu || nu == ign) continue;
          planes++;
          for (int sg = 1; sg >= -1; sg -= 2) {
            const int v = sg * (nu + 1);
            if (kind == 0) {
              const int p[3] = {v, -m, -v};
              for (int j = 0; j < 3; j++) t.steps[mu][n][j] = enc(p[j]);
              t.length[n] = 3;
              t.coeff[n++] = cp;
            } else {
              const int p[3][5] = {{m, v, -m, -m, -v}, {v, -m, -m, -v, m}, {v, v, -m, -v, -v}};
              for (int r = 0; r < 3; r++) {
                for (int j = 0; j < 5; j++) t.steps[mu][n][j] = enc(p[r][j]);
                t.length[n] = 5;
                t.coeff[n++] = cr;
              }
            }
          }
        }
      }
      t.n = n;
    }
    t.max_length = rect ? 5 : 3;
  }

  template <typename T>
  void fill_gauge_stout(GaugeStoutArgs<T> &a, const GaugeSmearRequest &rq, const void *const src[4], void *const dst[4])
  {
    SmearPaths t;
    const bool ovr = rq.type == B200_SMEAR_OVRIMP_STOUT;
    const double eps = ovr ? rq.coeff[1] : 0.0;
    smear_paths(t, rq.ign, ovr, ovr ? (5.0 - 2.0 * eps) / 3.0 : 1.0, -(1.0 - eps) / 12.0);
    int flat[4 * B200_GAUGE_MAX_PATHS * 5];
    for (int mu = 0; mu < 4; mu++)
      for (int i = 0; i < t.n; i++)
        for (int j = 0; j < t.max_length; j++) flat[(mu * t.n + i) * t.max_length + j] = j < t.length[i] ? t.steps[mu][i][j] : 0;
    GaugeForceRequest f {};
    for (int d = 0; d < 4; d++) {
      f.qdp[d] = src[d];
      f.X[d] = rq.X[d];
      a.out[d] = reinterpret_cast<T *>(dst[d]);
    }
    f.paths = flat;
    f.length = t.length;
    f.coeff = t.coeff;
    f.num_paths = t.n;
    f.max_length = t.max_length;
    f.eb3 = rq.coeff[0];
    fill_gauge_force(a.f, f);
    a.ign = rq.ign;
  }

  template <typename T> B2_HD void gauge_stout_site(const GaugeStoutArgs<T> &a, int x_cb, int parity, int mu)
  {
    Geom geo;
    geom_init(geo, a.f.g.X);
    int y[4];
    coords_from_cb(y, geo, x_cb, parity);
    T w[18], e[10], p[18], u[18], r[18];
    gauge_path_sum(w, a.f, y, mu); // rho Omega
#pragma unroll
    for (int k = 0; k < 10; k++) e[k] = 0;
    mom_sub_ta(e, w); // -rho TA(Omega) = rho TA(S U^+)
    mom_traceless(p, e, (T)1);
    su3_exp(w, p);
    load_link_ext(u, a.f.g, mu, y, 0, 0, 0, 0);
    su3_mul_op<false, false>(r, w, u);
    T *o = a.out[mu] + ((size_t)parity * a.f.g.volume_cb + x_cb) * 18;
#pragma unroll
    for (int k = 0; k < 18; k++) o[k] = r[k];
  }

  // ------------------------------------------------------------------ kernel 2: one APE or HYP level
  enum SmearLevel { kSmearApe = 0, kSmearHyp1 = 1, kSmearHyp2 = 2, kSmearHyp3 = 3 };

  template <typename T> struct SmearLevelArgs {
    CloverBuildArgs<T> g; // this step's thin links (g.u) and the lattice
    const T *dec;         // HYP levels 2 and 3: the decorated links of the level before
    T *dec_out;           // HYP level 1, and level 2 in 4-d: the decorated links written
    T *out[4];            // APE and the last HYP level: the smeared links
    T keep, c, tol;       // 1 - alpha, alpha / (number of staples), the projection's tolerance
    int level, ign, ndir;
  };

  // slot of the decorated link (mu, v), v != mu, among the links of the smeared directions
  template <typename T> B2_HD size_t dec_slot(const SmearLevelArgs<T> &a, int mu, int v)
  {
    return (size_t)(mu - (mu > a.ign)) * (a.ndir - 1) + v - (v > mu) - (v > a.ign);
  }

  template <typename T> B2_HD const T *dec_link(const SmearLevelArgs<T> &a, int mu, int v)
  {
    return a.dec + dec_slot(a, mu, v) * 2 * a.g.volume_cb * 18;
  }

  // s += the two staples of the link mu at y in the plane (mu, nu), its mu-links read from fm and its nu-links from fn
  // ([V][3][3][2] each): fn(y) fm(y + nu) fn(y + mu)^+ + fn(y - nu)^+ fm(y - nu) fn(y - nu + mu)
  template <typename T>
  B2_HD void plane_staple(T *s, const CloverBuildArgs<T> &g, const T *fm, const T *fn, const int *y, int mu, int nu)
  {
    T a[18], b[18], t[18];
    load_matrix_ext(a, fn, g, y, mu, 0, nu, 0);
    load_matrix_ext(b, fm, g, y, mu, 0, nu, 1);
    su3_mul_op<false, false>(t, a, b);
    load_matrix_ext(a, fn, g, y, mu, 1, nu, 0);
    su3_mul_op<false, true, true>(s, t, a);
    load_matrix_ext(a, fn, g, y, mu, 0, nu, -1);
    load_matrix_ext(b, fm, g, y, mu, 0, nu, -1);
    su3_mul_op<true, false>(t, a, b);
    load_matrix_ext(a, fn, g, y, mu, 1, nu, -1);
    su3_mul_op<false, false, true>(s, t, a);
  }

  // r = P[keep 1 + c s u^+] u
  template <typename T> B2_HD void smear_link(T *r, const SmearLevelArgs<T> &a, const T *s, const T *u)
  {
    T w[18], p[18];
    su3_mul_op<false, true>(w, s, u);
#pragma unroll
    for (int k = 0; k < 18; k++) w[k] = k % 8 == 0 ? fma_rn(a.c, w[k], a.keep) : mul_rn(a.c, w[k]);
    su3_project(p, w, a.tol);
    su3_mul_op<false, false>(r, p, u);
  }

  template <typename T> B2_HD void store_link(T *o, const T *r)
  {
#pragma unroll
    for (int k = 0; k < 18; k++) o[k] = r[k];
  }

  // APE: the staples of every smeared plane on the thin links.  HYP level 1: per plane v the decorated link from that
  // plane's thin staples.  Level 2: per excluded direction v (4-d; 3-d: v = ign, one output) the staples of the planes
  // rho != mu, v on the level-1 links decorated in the remaining plane sigma.  Level 3 (4-d): the staples of every plane nu
  // on the level-2 links of (mu excluding nu) and (nu excluding mu).
  template <typename T> B2_HD void gauge_smear_level_site(const SmearLevelArgs<T> &a, int x_cb, int parity, int mu)
  {
    Geom geo;
    geom_init(geo, a.g.X);
    int y[4];
    coords_from_cb(y, geo, x_cb, parity);
    const size_t site = (size_t)parity * a.g.volume_cb + x_cb, V = 2 * (size_t)a.g.volume_cb;
    T u[18], s[18], r[18];
    load_link_ext(u, a.g, mu, y, 0, 0, 0, 0);
    if (a.level == kSmearApe || a.level == kSmearHyp3) {
#pragma unroll
      for (int k = 0; k < 18; k++) s[k] = 0;
#pragma unroll 1
      for (int nu = 0; nu < 4; nu++) {
        if (nu == mu || nu == a.ign) continue;
        if (a.level == kSmearApe) plane_staple(s, a.g, a.g.u[mu], a.g.u[nu], y, mu, nu);
        else plane_staple(s, a.g, dec_link(a, mu, nu), dec_link(a, nu, mu), y, mu, nu);
      }
      smear_link(r, a, s, u);
      store_link(a.out[mu] + site * 18, r);
      return;
    }
#pragma unroll 1
    for (int v = 0; v < 4; v++) {
      if (v == mu || (a.level == kSmearHyp1 && v == a.ign) || (a.level == kSmearHyp2 && a.ign < 4 && v != a.ign)) continue;
#pragma unroll
      for (int k = 0; k < 18; k++) s[k] = 0;
      if (a.level == kSmearHyp1) {
        plane_staple(s, a.g, a.g.u[mu], a.g.u[v], y, mu, v);
      } else {
#pragma unroll 1
        for (int rho = 0; rho < 4; rho++) {
          if (rho == mu || rho == v || rho == a.ign) continue;
          const int sigma = 6 - mu - v - rho;
          plane_staple(s, a.g, dec_link(a, mu, sigma), dec_link(a, rho, sigma), y, mu, rho);
        }
      }
      smear_link(r, a, s, u);
      T *o = a.level == kSmearHyp2 && a.ign < 4 ? a.out[mu] + site * 18 : a.dec_out + (dec_slot(a, mu, v) * V + site) * 18;
      store_link(o, r);
    }
  }

  template <typename T>
  void fill_smear_level(SmearLevelArgs<T> &a, const GaugeSmearRequest &rq, int level, const void *const src[4], const T *dec,
                        T *dec_out, void *const dst[4], double alpha, int staples)
  {
    fill_lattice(a.g, src, rq.X);
    a.dec = dec;
    a.dec_out = dec_out;
    for (int d = 0; d < 4; d++) a.out[d] = reinterpret_cast<T *>(dst[d]);
    a.keep = (T)(1.0 - alpha);
    a.c = (T)(alpha / staples);
    a.tol = kProjectTol<T>;
    a.level = level;
    a.ign = rq.ign;
    a.ndir = rq.ign < 4 ? 3 : 4;
  }

  // ------------------------------------------------------------------ the launch sequence of both executors
  // step s reads src(s) and writes dst(s), ping-ponging between out and the scratch field as the flow's stages do
  inline FlowPlan smear_plan(const GaugeSmearRequest &rq)
  {
    FlowPlan p;
    p.stages = rq.n_steps;
    p.first_to_scratch = links_alias(rq.out, rq.in) ? true : ((p.stages - 1) & 1) == 1;
    return p;
  }

  // whether some step writes the scratch link field: every call but one step out of place
  inline bool smear_pingpong(const FlowPlan &p) { return p.first_to_scratch || p.stages > 1; }

  // Scratch, in link fields of [V][3][3][2]: the ping-pong field of the d smeared directions where a step writes it, then
  // for HYP the level-1 links (d (d - 1)) and in 4-d the level-2 links (12).
  inline size_t smear_scratch_links(const GaugeSmearRequest &rq)
  {
    const int d = rq.ign < 4 ? 3 : 4;
    return (smear_pingpong(smear_plan(rq)) ? d : 0) + (rq.type == B200_SMEAR_HYP ? d * (d - 1) + (d == 4 ? 12 : 0) : 0);
  }

  // Runs the smearing on executor x: x.stout(args, ndir) and x.level(args, ndir) launch a grid (blocks, ndir, parity),
  // x.copy(dst, src, bytes) copies device memory.  Each step is one launch (HYP: one per level); the links of the ignored
  // direction are never read (the scratch field has none) and are copied from in at the end.
  template <typename T, class Ex> int run_gauge_smear(const GaugeSmearRequest &rq, T *scratch, Ex &x)
  {
    const size_t L = (size_t)rq.X[0] * rq.X[1] * rq.X[2] * rq.X[3] * 18; // reals per link field
    const int ndir = rq.ign < 4 ? 3 : 4;
    const FlowPlan plan = smear_plan(rq);
    const bool pingpong = smear_pingpong(plan);
    void *tmp[4];
    for (int d = 0, k = 0; d < 4; d++) tmp[d] = pingpong && d != rq.ign ? scratch + (k++) * L : nullptr;
    T *d1 = scratch + (pingpong ? ndir : 0) * L, *d2 = d1 + ndir * (ndir - 1) * L;
    const void *src[4];
    for (int d = 0; d < 4; d++) src[d] = rq.in[d];
    int rc = 0;
    for (int s = 0; s < plan.stages && !rc; s++) {
      void *const *dst = plan.writes_scratch(s) ? tmp : rq.out;
      if (rq.type == B200_SMEAR_STOUT || rq.type == B200_SMEAR_OVRIMP_STOUT) {
        GaugeStoutArgs<T> a;
        fill_gauge_stout(a, rq, src, dst);
        rc = x.stout(a, ndir);
      } else if (rq.type == B200_SMEAR_APE) {
        SmearLevelArgs<T> a;
        fill_smear_level<T>(a, rq, kSmearApe, src, nullptr, nullptr, dst, rq.coeff[0], 2 * (ndir - 1));
        rc = x.level(a, ndir);
      } else {
        SmearLevelArgs<T> a;
        fill_smear_level<T>(a, rq, kSmearHyp1, src, nullptr, d1, dst, rq.coeff[2], 2);
        rc = x.level(a, ndir);
        if (!rc) {
          fill_smear_level<T>(a, rq, kSmearHyp2, src, d1, d2, dst, rq.coeff[1], 4);
          rc = x.level(a, ndir);
        }
        if (!rc && ndir == 4) {
          fill_smear_level<T>(a, rq, kSmearHyp3, src, d2, nullptr, dst, rq.coeff[0], 6);
          rc = x.level(a, ndir);
        }
      }
      for (int d = 0; d < 4; d++) src[d] = dst[d];
    }
    if (!rc && plan.ends_in_scratch())
      for (int d = 0; d < 4 && !rc; d++)
        if (d != rq.ign) rc = x.copy(rq.out[d], tmp[d], L * sizeof(T));
    if (!rc && rq.ign < 4 && rq.out[rq.ign] != rq.in[rq.ign]) rc = x.copy(rq.out[rq.ign], rq.in[rq.ign], L * sizeof(T));
    return rc;
  }

  // ------------------------------------------------------------------ entry point (executor E: the CUDA library or the twin)
  template <typename T> int launch_gauge_smear(const GaugeSmearRequest &rq); // inst_gauge_smear.cu

  template <class E>
  int gauge_smear(void *const out[4], const void *const in[4], const int X[4], int precision, int type, const double coeff[3],
                  int dir_ignore, int n_steps, void *stream)
  {
    if (int rc = check_gauge_smear(out, in, X, precision, type, coeff, dir_ignore, n_steps)) return rc;
    if (int rc = E::require_device()) return rc;
    GaugeSmearRequest rq {};
    for (int d = 0; d < 4; d++) {
      rq.out[d] = out[d];
      rq.in[d] = in[d];
      rq.X[d] = X[d];
    }
    rq.type = type;
    for (int i = 0; i < 3; i++) rq.coeff[i] = i < smear_coeff_count(type) ? coeff[i] : 0.0;
    rq.ign = dir_ignore < 0 ? 4 : dir_ignore;
    rq.n_steps = n_steps;
    rq.stream = stream;
    return precision == B200_DOUBLE ? E::template gauge_smear<double>(rq) : E::template gauge_smear<float>(rq);
  }

} // namespace b200
