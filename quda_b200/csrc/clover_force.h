// Clover fermion force: the momentum update of computeCloverForceQuda for the non-twisted Wilson-clover operator with
// asymmetric even-odd preconditioning (MATPCDAG_MATPC solutions, no determinant ratio).  Site code (B2_HD) shared by the
// CUDA kernels (inst_clover_force.cu) and the host twin, plus the argument validation and the entry-point body of
// b200_clover_force_accumulate.
//
// Reference behaviour reproduced (the reference's include/kernels/...):
//   clover_outer_product.cuh        hopping force  U_mu(x) sum_i c_i tr_spin[(1+g_mu) x_i(x+mu) p_i(x)^+
//                                                                         + (1-g_mu) p_i(x+mu) x_i(x)^+]
//   clover_sigma_outer_product.cuh  oprod_mu,nu = R - R^+,  R = sum_i eps_i[parity] tr_spin[sigma_nu,mu x_i p_i^+]
//   clover_trace.cuh                oprod_mu,nu += sigma_coeff tr_spin[sigma A^-1] on the tr log parity (chiral blocks)
//   clover_deriv.cuh                insertion of oprod_mu,nu at the four corners of the two leaves that hold U_mu(x)
//   momentum.cuh (updateMomentum)   mom -= TA(force), TA = traceless anti-Hermitian part
// Differences on purpose: TA is linear, so the hopping force and the derivative are each projected and subtracted from mom
// as soon as they are known and no [4][V] force field is written; A^-1 is recomputed in registers from the packed A by
// clover_build.h's Cholesky, so no inverse field is needed.  Only oprod goes through memory, because the derivative reads
// it at neighbouring sites.
//
// Field orders: spinors native (UKQCD basis, fp64 planes of 2 reals, fp32 planes of 4), full lattice, parity blocks of Vh
// sites; links QDP [4][V][3][3][2] as b200_compute_clover reads them (border 0); packed A [V][2][36]; mom [V][4][10]
// (the (01), (02), (12) complex entries, the three imaginary diagonals, one pad real: QUDA_ASQTAD_MOM_LINKS order);
// oprod [6][V][3][3][2].  Sites are parity-major everywhere.
#pragma once

#include "clover_build.h"

namespace b200
{

  // ------------------------------------------------------------------ request
  struct CloverForceRequest {
    void *mom;          // [V][4][10], accumulated
    const void *qdp[4]; // links U_mu, QDP order [V][3][3][2]
    const void *packed; // A, [V][2][36]
    int X[4];
    int n;                 // vectors
    const void *const *x;  // n full-lattice native spinors
    const void *const *p;  // n full-lattice native spinors
    const double *force_coeff; // [n]
    const double *eps;         // [n][2]: the sigma outer-product coefficient on even / odd sites
    double sigma_coeff;        // coefficient of tr[sigma A^-1]
    int trlog_parity;          // parity whose A^-1 enters the tr log force
    void *stream;
  };

  constexpr int kCloverForceThreads = 128;

  // ------------------------------------------------------------------ validation (shared by the library and the host twin)
  inline int check_clover_force(void *mom, const void *const qdp[4], const void *packed, const int X[4], int precision, int n,
                                const void *const *x, const void *const *p, const double *force_coeff, const double *eps,
                                double sigma_coeff, int trlog_parity)
  {
    const char *fn = "b200_clover_force_accumulate";
    if (!mom || !qdp || !packed || !x || !p || !force_coeff || !eps) return set_error(B200_ERR_INVALID, "%s: null argument", fn);
    if (n < 1 || n > B200_MAX_SHIFTS) return set_error(B200_ERR_INVALID, "%s: n=%d not in [1, %d]", fn, n, B200_MAX_SHIFTS);
    for (int d = 0; d < 4; d++)
      if (!qdp[d]) return set_error(B200_ERR_INVALID, "%s: qdp[%d] is NULL", fn, d);
    for (int i = 0; i < n; i++)
      if (!x[i] || !p[i]) return set_error(B200_ERR_INVALID, "%s: spinor pair %d is NULL", fn, i);
    if (int rc = check_clover_lattice(fn, X, precision)) return rc;
    if (trlog_parity != 0 && trlog_parity != 1) return set_error(B200_ERR_INVALID, "%s: trlog parity %d not in {0,1}", fn, trlog_parity);
    if (!std::isfinite(sigma_coeff)) return set_error(B200_ERR_INVALID, "%s: sigma_coeff is not finite", fn);
    for (int i = 0; i < n; i++)
      if (!std::isfinite(force_coeff[i]) || !std::isfinite(eps[2 * i]) || !std::isfinite(eps[2 * i + 1]))
        return set_error(B200_ERR_INVALID, "%s: coefficients of vector %d are not finite", fn, i);
    return 0;
  }

  // ------------------------------------------------------------------ kernel arguments
  template <typename T> struct CloverForceArgs {
    CloverBuildArgs<T> g; // links and lattice (border 0)
    T *mom;
    T *oprod;
    const T *packed;
    const T *x[B200_MAX_SHIFTS], *p[B200_MAX_SHIFTS];
    T force_coeff[B200_MAX_SHIFTS], eps[B200_MAX_SHIFTS][2];
    T sigma_coeff;
    int n, trlog_parity, volume_cb;
  };

  template <typename T> void fill_clover_force(CloverForceArgs<T> &a, const CloverForceRequest &rq, T *oprod)
  {
    CloverBuildRequest b {};
    for (int d = 0; d < 4; d++) {
      b.qdp[d] = rq.qdp[d];
      b.X[d] = rq.X[d];
    }
    fill_clover_build(a.g, b);
    a.mom = reinterpret_cast<T *>(rq.mom);
    a.oprod = oprod;
    a.packed = reinterpret_cast<const T *>(rq.packed);
    a.n = rq.n;
    for (int i = 0; i < rq.n; i++) {
      a.x[i] = reinterpret_cast<const T *>(rq.x[i]);
      a.p[i] = reinterpret_cast<const T *>(rq.p[i]);
      a.force_coeff[i] = (T)rq.force_coeff[i];
      a.eps[i][0] = (T)rq.eps[2 * i];
      a.eps[i][1] = (T)rq.eps[2 * i + 1];
    }
    a.sigma_coeff = (T)rq.sigma_coeff;
    a.trlog_parity = rq.trlog_parity;
    a.volume_cb = a.g.volume_cb;
  }

  // ------------------------------------------------------------------ site helpers
  template <typename T> using SpinorPrec = std::conditional_t<sizeof(T) == 8, PrecF64, PrecF32>;

  // the 24 reals (spin, colour, re/im) of native spinor f at (x_cb, parity)
  template <typename T> B2_HD void load_spinor(T *v, const T *f, int volume_cb, int x_cb, int parity)
  {
    SpinorView<SpinorPrec<T>> s {const_cast<T *>(f) + (size_t)parity * volume_cb * 24, nullptr, volume_cb};
    s.load(v, x_cb);
  }

  // r += c tr_spin[a b^+]: r(j,k) += c sum_s a(s,j) conj(b(s,k))  (outerProdSpinTrace)
  template <typename T> B2_HD void outer_spin_trace_acc(T *r, const T *a, const T *b, T c)
  {
#pragma unroll
    for (int j = 0; j < 3; j++) {
#pragma unroll
      for (int k = 0; k < 3; k++) {
        T re = 0, im = 0;
#pragma unroll
        for (int s = 0; s < 4; s++) {
          const T ar = a[(s * 3 + j) * 2], ai = a[(s * 3 + j) * 2 + 1], br = b[(s * 3 + k) * 2], bi = b[(s * 3 + k) * 2 + 1];
          re = fma_rn(ar, br, re);
          re = fma_rn(ai, bi, re);
          im = fma_rn(ai, br, im);
          im = fma_rn(-ar, bi, im);
        }
        r[(j * 3 + k) * 2] = fma_rn(c, re, r[(j * 3 + k) * 2]);
        r[(j * 3 + k) * 2 + 1] = fma_rn(c, im, r[(j * 3 + k) * 2 + 1]);
      }
    }
  }

  // mom -= TA(f) for one link: TA(f) = (f - f^+)/2 - i Im tr(f)/3, then the diagonal is made traceless again as
  // updateMomentum's final projection does
  template <typename T> B2_HD void mom_sub_ta(T *m, const T *f)
  {
    constexpr int od[3][2] = {{0, 1}, {0, 2}, {1, 2}};
#pragma unroll
    for (int n = 0; n < 3; n++) {
      const int ij = (od[n][0] * 3 + od[n][1]) * 2, ji = (od[n][1] * 3 + od[n][0]) * 2;
      m[2 * n] -= (f[ij] - f[ji]) * (T)0.5;
      m[2 * n + 1] -= (f[ij + 1] + f[ji + 1]) * (T)0.5;
    }
    const T tr = (f[1] + f[9] + f[17]) / (T)3;
    T d[3];
#pragma unroll
    for (int k = 0; k < 3; k++) d[k] = m[6 + k] - (f[(k * 4) * 2 + 1] - tr);
    const T md = (d[0] + d[1] + d[2]) / (T)3;
#pragma unroll
    for (int k = 0; k < 3; k++) m[6 + k] = d[k] - md;
  }

  template <typename T> B2_HD T *mom_link(const CloverForceArgs<T> &a, int x_cb, int parity, int mu)
  {
    return a.mom + (((size_t)parity * a.volume_cb + x_cb) * 4 + mu) * 10;
  }

  // ------------------------------------------------------------------ kernel 1: hopping force -> mom
  // The x term uses the projector of the forward hop of D^+, the p term that of D (dslash_site.h hop_sign).
  template <typename T> B2_HD void clover_hop_force_site(const CloverForceArgs<T> &a, int x_cb, int parity, int mu)
  {
    Geom geo;
    geom_init(geo, a.g.X);
    int y[4];
    coords_from_cb(y, geo, x_cb, parity);
    const int nb = neighbor_cb<true>(y, geo, mu);
    T r[18];
#pragma unroll
    for (int i = 0; i < 18; i++) r[i] = 0;
#pragma unroll 1
    for (int i = 0; i < a.n; i++) {
#pragma unroll
      for (int term = 0; term < 2; term++) {
        const T *nbr_f = term ? a.p[i] : a.x[i], *loc_f = term ? a.x[i] : a.p[i];
        const int sign = term ? hop_sign<false, true>() : hop_sign<true, true>();
        T v[24], h[12], w[24];
        load_spinor(v, nbr_f, a.volume_cb, nb, 1 - parity);
        project(h, v, mu, sign);
#pragma unroll
        for (int k = 0; k < 24; k++) w[k] = 0;
        reconstruct_add(w, h, mu, sign);
        load_spinor(v, loc_f, a.volume_cb, x_cb, parity);
        outer_spin_trace_acc(r, w, v, a.force_coeff[i]);
      }
    }
    T u[18], f[18];
    load_link_ext(u, a.g, mu, y, 0, 0, 0, 0);
    su3_mul_op<false, false>(f, u, r);
    mom_sub_ta(mom_link(a, x_cb, parity, mu), f);
  }

  // ------------------------------------------------------------------ kernel 2: sigma outer product + sigma trace -> oprod
  // sigma_nu,mu = gamma_nu gamma_mu of plane p (plane_map order) in the UKQCD basis: (sigma v)(s) = w(s) v(src(s)), weight
  // codes as add_weighted's (0: +1, 1: -1, 2: +i, 3: -i)
  struct SigmaMap {
    int src[4], w[4];
  };
  B2_HD constexpr SigmaMap sigma_map(int p)
  {
    switch (p) {
    case 0: return {{0, 1, 2, 3}, {2, 3, 2, 3}}; // sigma_0,1
    case 1: return {{1, 0, 3, 2}, {1, 0, 1, 0}}; // sigma_0,2
    case 2: return {{1, 0, 3, 2}, {2, 2, 2, 2}}; // sigma_1,2
    case 3: return {{3, 2, 1, 0}, {3, 3, 3, 3}}; // sigma_0,3
    case 4: return {{3, 2, 1, 0}, {1, 0, 1, 0}}; // sigma_1,3
    default: return {{2, 3, 0, 1}, {3, 2, 3, 2}}; // sigma_2,3
    }
  }

  // tr_spin[sigma A^-1] of plane p from the two chiral blocks of A^-1 (clover_trace.cuh): a phase times a signed sum of the
  // 3x3 quadrants UL, LR, UR, LL of each block; weights [quadrant][chirality] in {-1, 0, +1}
  struct TraceMap {
    int phase; // add_weighted code
    int w[4][2];
  };
  B2_HD constexpr TraceMap trace_map(int p)
  {
    switch (p) {
    case 0: return {2, {{-1, -1}, {1, 1}, {0, 0}, {0, 0}}};  // i (LR0 + LR1 - UL0 - UL1)
    case 1: return {0, {{0, 0}, {0, 0}, {1, 1}, {-1, -1}}};  // UR0 - LL0 + UR1 - LL1
    case 2: return {3, {{0, 0}, {0, 0}, {1, 1}, {1, 1}}};    // -i (UR0 + LL0 + UR1 + LL1)
    case 3: return {2, {{0, 0}, {0, 0}, {1, -1}, {1, -1}}};  // i (UR0 + LL0 - UR1 - LL1)
    case 4: return {0, {{0, 0}, {0, 0}, {1, -1}, {-1, 1}}};  // UR0 - LL0 - UR1 + LL1
    default: return {2, {{1, -1}, {-1, 1}, {0, 0}, {0, 0}}}; // i (UL0 - LR0 - UL1 + LR1)
    }
  }

  // entry (i, j) of a Hermitian 6x6 block in packed order
  template <typename T> B2_HD void hermitian_entry(T &re, T &im, const T *h, int i, int j)
  {
    if (i == j) {
      re = h[i];
      im = 0;
    } else if (i > j) {
      re = h[tri_idx(i, j)];
      im = h[tri_idx(i, j) + 1];
    } else {
      re = h[tri_idx(j, i)];
      im = -h[tri_idx(j, i) + 1];
    }
  }

  // r += c tr_spin[sigma A^-1] of plane p at packed site `site`
  template <int p, typename T> B2_HD void add_sigma_trace(T *r, const CloverForceArgs<T> &a, size_t site, T c)
  {
    T inv[2][36];
#pragma unroll
    for (int ch = 0; ch < 2; ch++) clover_block_invert<T>(inv[ch], a.packed + site * 72 + 36 * ch);
    constexpr TraceMap m = trace_map(p);
    constexpr int off[4][2] = {{0, 0}, {3, 3}, {0, 3}, {3, 0}}; // UL, LR, UR, LL: row / column offsets
#pragma unroll
    for (int j = 0; j < 3; j++) {
#pragma unroll
      for (int k = 0; k < 3; k++) {
        T sr = 0, si = 0;
#pragma unroll
        for (int q = 0; q < 4; q++) {
#pragma unroll
          for (int ch = 0; ch < 2; ch++) {
            if (!m.w[q][ch]) continue;
            T er, ei;
            hermitian_entry(er, ei, inv[ch], j + off[q][0], k + off[q][1]);
            add_weighted(sr, si, er, ei, m.w[q][ch] > 0 ? 0 : 1);
          }
        }
        T tr = 0, ti = 0;
        add_weighted(tr, ti, sr, si, m.phase);
        r[(j * 3 + k) * 2] = fma_rn(c, tr, r[(j * 3 + k) * 2]);
        r[(j * 3 + k) * 2 + 1] = fma_rn(c, ti, r[(j * 3 + k) * 2 + 1]);
      }
    }
  }

  // plane p is a template parameter so that the spin maps index registers, not local memory
  template <int p, typename T> B2_HD void clover_sigma_site(const CloverForceArgs<T> &a, int x_cb, int parity)
  {
    constexpr SigmaMap s = sigma_map(p);
    T r[18];
#pragma unroll
    for (int i = 0; i < 18; i++) r[i] = 0;
#pragma unroll 1
    for (int i = 0; i < a.n; i++) {
      T v[24], w[24];
      load_spinor(v, a.x[i], a.volume_cb, x_cb, parity);
#pragma unroll
      for (int sp = 0; sp < 4; sp++) {
#pragma unroll
        for (int c = 0; c < 3; c++) {
          T re = 0, im = 0;
          add_weighted(re, im, v[(s.src[sp] * 3 + c) * 2], v[(s.src[sp] * 3 + c) * 2 + 1], s.w[sp]);
          w[(sp * 3 + c) * 2] = re;
          w[(sp * 3 + c) * 2 + 1] = im;
        }
      }
      load_spinor(v, a.p[i], a.volume_cb, x_cb, parity);
      outer_spin_trace_acc(r, w, v, a.eps[i][parity]);
    }
    T o[18]; // R - R^+
#pragma unroll
    for (int j = 0; j < 3; j++) {
#pragma unroll
      for (int k = 0; k < 3; k++) {
        o[(j * 3 + k) * 2] = r[(j * 3 + k) * 2] - r[(k * 3 + j) * 2];
        o[(j * 3 + k) * 2 + 1] = r[(j * 3 + k) * 2 + 1] + r[(k * 3 + j) * 2 + 1];
      }
    }
    const size_t site = (size_t)parity * a.volume_cb + x_cb;
    if (parity == a.trlog_parity) add_sigma_trace<p>(o, a, site, a.sigma_coeff);
    T *out = a.oprod + ((size_t)p * 2 * a.volume_cb + site) * 18;
#pragma unroll
    for (int i = 0; i < 18; i++) out[i] = o[i];
  }

  // ------------------------------------------------------------------ kernel 3: clover derivative -> mom
  // Position after the first k links of leaf `leaf` (kLeaf), as (steps along mu, steps along nu); k = 0 is x itself
  template <int leaf, int k, int along_nu> B2_HD constexpr int leaf_corner()
  {
    if constexpr (k == 0) {
      return 0;
    } else {
      constexpr LeafLink L = kLeaf[leaf][k - 1];
      return (along_nu ? L.dnu : L.dmu) + (!L.dag && L.dir == along_nu ? 1 : 0); // U: site -> site + dir; U^+ returns to site
    }
  }

  template <typename T> B2_HD void su3_copy_dag(T *r, const T *a)
  {
#pragma unroll
    for (int i = 0; i < 3; i++) {
#pragma unroll
      for (int j = 0; j < 3; j++) {
        r[(i * 3 + j) * 2] = a[(j * 3 + i) * 2];
        r[(i * 3 + j) * 2 + 1] = -a[(j * 3 + i) * 2 + 1];
      }
    }
  }

  // f (+/-)= sum_k l_0 .. l_{k-1} O(corner k) l_k .. l_3 over the four corners of leaf 0 (k = 1..4, the leaf starts with
  // U_mu(x)) or leaf 2 (k = 0..3, it ends with U_mu(x)^+), O = oprod plane t.  Evaluated from the last link backwards:
  // S_j = l_j S_{j+1}, Y_j = l_j Y_{j+1} + [k = j inserted] O_j S_j, so every link is loaded once.
  template <int leaf, typename T>
  B2_HD void leaf_insertions(T *f, const CloverForceArgs<T> &a, const int *y, int mu, int nu, int t, bool subtract)
  {
    static_assert(leaf == 0 || leaf == 2, "only leaves 0 and 2 contain U_mu(x)");
    const T *O = a.oprod + (size_t)t * 2 * a.volume_cb * 18;
    T l[18], S[18], Y[18], q[18], tmp[18];
    auto corner = [&](T *o, auto kc) {
      constexpr int k = decltype(kc)::value;
      load_matrix_ext(o, O, a.g, y, mu, leaf_corner<leaf, k, 0>(), nu, leaf_corner<leaf, k, 1>());
    };
    // j = 3
    leaf_link<leaf, 3>(l, a.g, y, mu, nu);
    constexpr bool d3 = kLeaf[leaf][3].dag;
    corner(q, std::integral_constant<int, 3>());
    su3_mul_op<false, d3>(Y, q, l); // O_3 l_3
    if (leaf == 0) {
      corner(q, std::integral_constant<int, 4>());
      su3_mul_op<d3, false, true>(Y, l, q); // + l_3 O_4
    }
    if (d3) su3_copy_dag(S, l);
    else
      for (int i = 0; i < 18; i++) S[i] = l[i];
    // j = 2, 1, 0
    auto step = [&](auto jc) {
      constexpr int j = decltype(jc)::value;
      constexpr bool dj = kLeaf[leaf][j].dag;
      leaf_link<leaf, j>(l, a.g, y, mu, nu);
      su3_mul_op<dj, false>(tmp, l, Y);
#pragma unroll
      for (int i = 0; i < 18; i++) Y[i] = tmp[i];
      if (j > 0 || leaf == 2) {
        su3_mul_op<dj, false>(tmp, l, S);
#pragma unroll
        for (int i = 0; i < 18; i++) S[i] = tmp[i];
        corner(q, jc);
        su3_mul_op<false, false, true>(Y, q, S);
      }
    };
    step(std::integral_constant<int, 2>());
    step(std::integral_constant<int, 1>());
    step(std::integral_constant<int, 0>());
#pragma unroll
    for (int i = 0; i < 18; i++) f[i] = subtract ? f[i] - Y[i] : f[i] + Y[i];
  }

  template <typename T> B2_HD void clover_sigma_site(const CloverForceArgs<T> &a, int x_cb, int parity, int p)
  {
    switch (p) {
    case 0: clover_sigma_site<0>(a, x_cb, parity); break;
    case 1: clover_sigma_site<1>(a, x_cb, parity); break;
    case 2: clover_sigma_site<2>(a, x_cb, parity); break;
    case 3: clover_sigma_site<3>(a, x_cb, parity); break;
    case 4: clover_sigma_site<4>(a, x_cb, parity); break;
    default: clover_sigma_site<5>(a, x_cb, parity); break;
    }
  }

  template <typename T> B2_HD void clover_deriv_site(const CloverForceArgs<T> &a, int x_cb, int parity, int mu)
  {
    Geom geo;
    geom_init(geo, a.g.X);
    int y[4];
    coords_from_cb(y, geo, x_cb, parity);
    T f[18];
#pragma unroll
    for (int i = 0; i < 18; i++) f[i] = 0;
#pragma unroll 1
    for (int nu = 0; nu < 4; nu++) {
      if (nu == mu) continue;
      const int hi = mu > nu ? mu : nu, lo = mu > nu ? nu : mu;
      const int t = (hi - 1) * hi / 2 + lo; // plane_map order
      // the upper leaf enters with - for nu < mu, the lower one with the opposite sign (clover_deriv.cuh)
      leaf_insertions<0>(f, a, y, mu, nu, t, nu < mu);
      leaf_insertions<2>(f, a, y, mu, nu, t, !(nu < mu));
    }
    mom_sub_ta(mom_link(a, x_cb, parity, mu), f);
  }

  // ------------------------------------------------------------------ entry point (executor E: the CUDA library or the twin)
  template <typename T> int launch_clover_force(const CloverForceRequest &rq); // inst_clover_force.cu

  template <class E>
  int clover_force_accumulate(void *mom, const void *const qdp[4], const void *packed, const int X[4], int precision, int n,
                              const void *const *x, const void *const *p, const double *force_coeff, const double *eps,
                              double sigma_coeff, int trlog_parity, void *stream)
  {
    if (int rc = check_clover_force(mom, qdp, packed, X, precision, n, x, p, force_coeff, eps, sigma_coeff, trlog_parity)) return rc;
    if (int rc = E::require_device()) return rc;
    CloverForceRequest rq;
    rq.mom = mom;
    for (int d = 0; d < 4; d++) {
      rq.qdp[d] = qdp[d];
      rq.X[d] = X[d];
    }
    rq.packed = packed;
    rq.n = n;
    rq.x = x;
    rq.p = p;
    rq.force_coeff = force_coeff;
    rq.eps = eps;
    rq.sigma_coeff = sigma_coeff;
    rq.trlog_parity = trlog_parity;
    rq.stream = stream;
    return precision == B200_DOUBLE ? E::template clover_force<double>(rq) : E::template clover_force<float>(rq);
  }

} // namespace b200
