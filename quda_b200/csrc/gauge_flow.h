// Gradient flow of a gauge field and its observables: Lüscher's RK3 integration of dV/dt = Z(V) V for the action given as
// a gauge-force path table, and the clover energy density and topological charge.  Site code (B2_HD) shared by the CUDA
// kernels (inst_gauge_flow.cu) and the host twin, plus the argument validation and the entry-point bodies of
// b200_gauge_flow / b200_gauge_observables.
//
// Reference behaviour reproduced:
//   include/kernels/gauge_wilson_flow.cuh:36-43,53-86   flow generator Z_mu(x) = -TA(Omega_mu(x)), Omega = U_mu(x) sum_i c_i
//                                                       path_i(x) (the gauge force's product); Wilson: the plaquette
//                                                       staples with c = 1, Symanzik: plaquette 5/3 and rectangle -1/12.
//                                                       This is the reference's exp(AH(staple U^+)) with its sign.
//   include/kernels/gauge_wilson_flow.cuh:88-174        RK3 of arXiv:1006.4518 App. C with Z_i = eps Z(W_i):
//                                                       W1 = exp(Z0 / 4) W0, W2 = exp(8/9 Z1 - 17/36 Z0) W1,
//                                                       W3 = exp(3/4 Z2 - 8/9 Z1 + 17/36 Z0) W2
//   include/kernels/gauge_qcharge.cuh:38-81,            F_p = (Q_p - Q_p^+) / 8 from the four clover leaves, planes in
//   include/kernels/field_strength_tensor.cuh:56-177,   plane_map order F10, F20, F21, F30, F31, F32; E_spatial / E_temporal
//   lib/gauge_qcharge.cu:45-47                          = sum of -Re tr(Fhat_p^2) over the planes with mu < 3 / mu = 3 over
//                                                       V (Fhat: F without its trace), E_total their sum;
//                                                       q(x) = -1/(4 pi^2) Re (tr F0 F5 - tr F1 F4 + tr F2 F3) on F itself
// Differences on purpose: one kernel per RK3 stage does the staple walk, the accumulator update, the exponential and the
// link product (the reference's staple kernel and update are one too, but it stores Z as a full matrix); the accumulator
// is the 10-real mom layout [V][4][10]; the sums are the fixed-order two-stage sums of gauge.h, so repeated calls are
// bit-identical.
//
// Field orders as gauge.h: links QDP [4][V][3][3][2] (boundary signs included), parity-major sites.
#pragma once

#include "gauge.h"

namespace b200
{

  // ------------------------------------------------------------------ requests
  struct GaugeFlowRequest {
    void *out[4];
    const void *in[4];
    int X[4];
    const int *paths; // [4][num_paths][max_length]
    const int *length;
    const double *coeff;
    int num_paths, max_length;
    double epsilon;
    int n_steps;
    void *stream;
  };

  struct GaugeObsRequest {
    const void *qdp[4];
    double *density; // device [V] or nullptr
    int X[4];
    void *stream;
  };

  // ------------------------------------------------------------------ validation (shared by the library and the host twin)
  inline int check_gauge_flow(void *const out[4], const void *const in[4], const int X[4], int precision, const int *paths,
                              const int *length, const double *coeff, int num_paths, int max_length, double epsilon,
                              int n_steps)
  {
    const char *fn = "b200_gauge_flow";
    if (!out) return set_error(B200_ERR_INVALID, "%s: null argument", fn);
    for (int d = 0; d < 4; d++)
      if (!out[d]) return set_error(B200_ERR_INVALID, "%s: output direction %d is NULL", fn, d);
    if (int rc = check_links(fn, in)) return rc;
    if (int rc = check_clover_lattice(fn, X, precision)) return rc;
    if (int rc = check_gauge_paths(fn, paths, length, coeff, num_paths, max_length)) return rc;
    if (!std::isfinite(epsilon)) return set_error(B200_ERR_INVALID, "%s: epsilon is not finite", fn);
    if (n_steps < 1) return set_error(B200_ERR_INVALID, "%s: n_steps=%d must be at least 1", fn, n_steps);
    return 0;
  }

  inline int check_gauge_observables(const double *energy, const double *qcharge, const void *const qdp[4], const int X[4],
                                     int precision)
  {
    const char *fn = "b200_gauge_observables";
    if (!energy || !qcharge) return set_error(B200_ERR_INVALID, "%s: null argument", fn);
    if (int rc = check_links(fn, qdp)) return rc;
    return check_clover_lattice(fn, X, precision);
  }

  // ------------------------------------------------------------------ kernel 1: one RK3 stage
  // E = alpha Z + beta A with Z = -eps TA(Omega) (f.eb3 = eps, A = f.mom), A <- E on stages 1 and 2, out = exp(gamma E) U
  template <typename T> struct GaugeFlowArgs {
    GaugeForceArgs<T> f; // links of this stage's input (f.g), the path table, eps (f.eb3), the accumulator (f.mom)
    T *out[4];
    T alpha, beta, gamma;
    int read_acc, store_acc;
  };
  static_assert(sizeof(GaugeFlowArgs<double>) <= 4096, "the gauge flow arguments must fit the kernel parameter block");

  // (alpha, beta, gamma) of RK3 stage 0, 1, 2
  constexpr double kFlowStage[3][3] = {{1.0, 0.0, 0.25}, {8.0 / 9, -17.0 / 36, 1.0}, {0.75, -1.0, 1.0}};

  // the stages of one call, as both executors run them: stage s reads src(s) and writes dst(s), ping-ponging between out
  // and one scratch field.  The first stage reads in; it must not write out when out is in (its neighbours still read in),
  // otherwise the first destination is chosen so that the last stage writes out.
  struct FlowPlan {
    int stages;
    bool first_to_scratch;
    B2_HD bool writes_scratch(int s) const { return ((s & 1) == 0) == first_to_scratch; }
    bool ends_in_scratch() const { return writes_scratch(stages - 1); }
  };

  inline bool links_alias(void *const out[4], const void *const in[4])
  {
    for (int d = 0; d < 4; d++)
      for (int e = 0; e < 4; e++)
        if (out[d] == in[e]) return true;
    return false;
  }

  inline FlowPlan flow_plan(const GaugeFlowRequest &rq)
  {
    FlowPlan p;
    p.stages = 3 * rq.n_steps;
    const bool last_even = ((p.stages - 1) & 1) == 0;
    p.first_to_scratch = links_alias(rq.out, rq.in) ? true : !last_even;
    return p;
  }

  // the arguments of stage s: src / dst are the link fields [4] it reads and writes, acc the accumulator [V][4][10]
  template <typename T>
  void fill_flow_stage(GaugeFlowArgs<T> &a, const GaugeFlowRequest &rq, int s, const void *const src[4], void *const dst[4], void *acc)
  {
    GaugeForceRequest f {};
    f.mom = acc;
    for (int d = 0; d < 4; d++) {
      f.qdp[d] = src[d];
      f.X[d] = rq.X[d];
      a.out[d] = reinterpret_cast<T *>(dst[d]);
    }
    f.paths = rq.paths;
    f.length = rq.length;
    f.coeff = rq.coeff;
    f.num_paths = rq.num_paths;
    f.max_length = rq.max_length;
    f.eb3 = rq.epsilon;
    fill_gauge_force(a.f, f);
    const int k = s % 3;
    a.alpha = (T)kFlowStage[k][0];
    a.beta = (T)kFlowStage[k][1];
    a.gamma = (T)kFlowStage[k][2];
    a.read_acc = k != 0; // the accumulator is uninitialised before the first stage, and 0 * NaN is NaN
    a.store_acc = k != 2;
  }

  template <typename T> B2_HD void gauge_flow_site(const GaugeFlowArgs<T> &a, int x_cb, int parity, int mu)
  {
    Geom geo;
    geom_init(geo, a.f.g.X);
    int y[4];
    coords_from_cb(y, geo, x_cb, parity);
    T w[18], e[10];
    gauge_path_sum(w, a.f, y, mu); // eps Omega
#pragma unroll
    for (int k = 0; k < 10; k++) e[k] = 0;
    mom_sub_ta(e, w); // Z = -eps TA(Omega)
    T *acc = mom_at(a.f.mom, a.f.g.volume_cb, x_cb, parity, mu);
    if (a.read_acc) {
#pragma unroll
      for (int k = 0; k < 9; k++) e[k] = fma_rn(a.beta, acc[k], mul_rn(a.alpha, e[k]));
    } else {
#pragma unroll
      for (int k = 0; k < 9; k++) e[k] = mul_rn(a.alpha, e[k]);
    }
    if (a.store_acc) {
#pragma unroll
      for (int k = 0; k < 9; k++) acc[k] = e[k];
    }
    T p[18], u[18], r[18];
    mom_traceless(p, e, (T)1);
#pragma unroll
    for (int k = 0; k < 18; k++) p[k] = mul_rn(a.gamma, p[k]);
    su3_exp(w, p);
    load_link_ext(u, a.f.g, mu, y, 0, 0, 0, 0);
    su3_mul_op<false, false>(r, w, u);
    T *o = a.out[mu] + ((size_t)parity * a.f.g.volume_cb + x_cb) * 18;
#pragma unroll
    for (int k = 0; k < 18; k++) o[k] = r[k];
  }

  // ------------------------------------------------------------------ kernel 2: energy density and topological charge
  // Re tr(A B) of two 3x3 complex matrices: the products in T, the sum in double
  template <typename T> B2_HD double re_tr_mul(const T *a, const T *b)
  {
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < 3; i++) {
#pragma unroll
      for (int j = 0; j < 3; j++) {
        const int ij = (i * 3 + j) * 2, ji = (j * 3 + i) * 2;
        s += (double)fma_rn(a[ij], b[ji], -mul_rn(a[ij + 1], b[ji + 1]));
      }
    }
    return s;
  }

  // F = (Q - Q^+) / 8 of plane p at y (Q the four clover leaves, summed as add_plane does), and -Re tr(Fhat^2)
  template <typename T> B2_HD double field_strength_plane(T *F, const CloverBuildArgs<T> &a, const int *y, int p)
  {
    const PlaneMap m = plane_map(p);
    T q[18];
#pragma unroll 1
    for (int leaf = 0; leaf < 4; leaf++) {
      switch (leaf) {
      case 0: leaf_product<0>(q, a, y, m.mu, m.nu); break;
      case 1: leaf_product<1>(q, a, y, m.mu, m.nu); break;
      case 2: leaf_product<2>(q, a, y, m.mu, m.nu); break;
      default: leaf_product<3>(q, a, y, m.mu, m.nu); break;
      }
    }
#pragma unroll
    for (int i = 0; i < 3; i++) {
#pragma unroll
      for (int j = 0; j < 3; j++) {
        const int ij = (i * 3 + j) * 2, ji = (j * 3 + i) * 2;
        F[ij] = mul_rn(q[ij] - q[ji], (T)0.125);
        F[ij + 1] = mul_rn(q[ij + 1] + q[ji + 1], (T)0.125);
      }
    }
    T h[18]; // Fhat = F - tr(F) / 3 (tr F is imaginary: the real diagonal of Q - Q^+ is exactly zero)
#pragma unroll
    for (int k = 0; k < 18; k++) h[k] = F[k];
    const T ti = (F[1] + F[9] + F[17]) / (T)3;
#pragma unroll
    for (int k = 0; k < 3; k++) h[k * 8 + 1] = F[k * 8 + 1] - ti;
    return -re_tr_mul(h, h);
  }

  // E_spatial, E_temporal (before the 1 / V) and q(x) at (x_cb, parity)
  constexpr double kQNorm = -1.0 / (4.0 * 3.14159265358979323846 * 3.14159265358979323846);
  template <typename T>
  B2_HD void gauge_obs_site(const CloverBuildArgs<T> &a, int x_cb, int parity, double &sp, double &tm, double &q)
  {
    Geom geo;
    geom_init(geo, a.X);
    int y[4];
    coords_from_cb(y, geo, x_cb, parity);
    sp = 0.0;
    tm = 0.0;
    double t = 0.0;
    // the charge pairs (F0, F5), (F1, F4), (F2, F3) with signs +, -, +: two planes' F at a time
#pragma unroll 1
    for (int i = 0; i < 3; i++) {
      T Fa[18], Fb[18];
      sp += field_strength_plane(Fa, a, y, i);    // planes 0..2: mu < 3
      tm += field_strength_plane(Fb, a, y, 5 - i); // planes 3..5: mu = 3
      const double c = re_tr_mul(Fa, Fb);
      t = i == 1 ? t - c : t + c;
    }
    q = mul_rn(kQNorm, t);
  }

  // the host's last step of b200_gauge_observables, from the per-group device sums g[kind][parity]
  inline void gauge_obs_total(double energy[3], double *qcharge, const double g[6], const int X[4])
  {
    const double V = (double)X[0] * X[1] * X[2] * X[3];
    energy[1] = (g[0] + g[1]) / V;
    energy[2] = (g[2] + g[3]) / V;
    energy[0] = energy[1] + energy[2];
    *qcharge = g[4] + g[5];
  }

  // ------------------------------------------------------------------ entry points (executor E: the CUDA library or the twin)
  template <typename T> int launch_gauge_flow(const GaugeFlowRequest &rq);                  // inst_gauge_flow.cu
  template <typename T> int launch_gauge_observables(const GaugeObsRequest &rq, double g[6]); // inst_gauge_flow.cu, synchronises

  template <class E>
  int gauge_flow(void *const out[4], const void *const in[4], const int X[4], int precision, const int *paths, const int *length,
                 const double *coeff, int num_paths, int max_length, double epsilon, int n_steps, void *stream)
  {
    if (int rc = check_gauge_flow(out, in, X, precision, paths, length, coeff, num_paths, max_length, epsilon, n_steps)) return rc;
    if (int rc = E::require_device()) return rc;
    GaugeFlowRequest rq;
    for (int d = 0; d < 4; d++) {
      rq.out[d] = out[d];
      rq.in[d] = in[d];
      rq.X[d] = X[d];
    }
    rq.paths = paths;
    rq.length = length;
    rq.coeff = coeff;
    rq.num_paths = num_paths;
    rq.max_length = max_length;
    rq.epsilon = epsilon;
    rq.n_steps = n_steps;
    rq.stream = stream;
    return precision == B200_DOUBLE ? E::template gauge_flow<double>(rq) : E::template gauge_flow<float>(rq);
  }

  template <class E>
  int gauge_observables(double energy[3], double *qcharge, double *density, const void *const qdp[4], const int X[4],
                        int precision, void *stream)
  {
    if (int rc = check_gauge_observables(energy, qcharge, qdp, X, precision)) return rc;
    if (int rc = E::require_device()) return rc;
    GaugeObsRequest rq {};
    for (int d = 0; d < 4; d++) {
      rq.qdp[d] = qdp[d];
      rq.X[d] = X[d];
    }
    rq.density = density;
    rq.stream = stream;
    double g[6];
    const int rc = precision == B200_DOUBLE ? E::template gauge_observables<double>(rq, g)
                                            : E::template gauge_observables<float>(rq, g);
    if (!rc) gauge_obs_total(energy, qcharge, g, X);
    return rc;
  }

} // namespace b200
