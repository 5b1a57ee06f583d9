// Clover term from the gauge links: A = 1 + kappa c_sw sum_{mu<nu} sigma_mu,nu F_mu,nu per chiral block, its inverse by
// Cholesky and log det A.  Site code (B2_HD) shared by the CUDA kernels (inst_clover_build.cu) and the host twin, plus the
// argument validation and the entry-point bodies of b200_compute_clover / b200_clover_invert_packed.
//
// Reference behaviour reproduced (the reference's include/...):
//   kernels/field_strength_tensor.cuh:40-178  four clover leaves per (mu, nu), F = (Q - Q^dagger) / 8 (no trace
//                                             subtraction), planes F10, F20, F21, F30, F31, F32
//   kernels/clover_compute.cuh:60-124         chiral blocks from F (block1 = i c (F0 -+ F5), block2 = c (F1 +- F4 - i (F2 -+ F3)))
//   kernels/clover_invert.cuh:44-84           Cholesky of each block (double for fp64 / fp32), tr log A = 2 sum log L_jj per
//                                             parity
// Differences on purpose: A is linear in F, so every plane's F is added into the block accumulators as soon as it is known
// and no Fmunu field is written to memory; the output is the packed host order [2 Vh][2][36] (A itself; b200_copy_clover
// halves it into the native layout).  Every product is an explicit fma_rn / mul_rn so that the CUDA kernels and the host
// twin round identically.
#pragma once

#include <cmath>

#include "launch.h"

namespace b200
{

  // ------------------------------------------------------------------ requests
  struct CloverBuildRequest {
    const void *qdp[4]; // links U_mu on the extended lattice, QDP order [2 Vh_e][3][3][2]
    void *packed;       // out: [2 Vh][2][36]
    int X[4], border[4];
    double coeff; // kappa * c_sw
    void *stream;
  };

  struct CloverInvertRequest {
    void *inv;          // out: A^-1 in packed order (nullptr: tr log only)
    const void *packed; // A in packed order
    double *trlog;      // out (host): per-parity sums of log det A
    int X[4];
    void *stream;
  };

  constexpr int kCloverBuildThreads = 128; // threads per CTA of both kernels (the trlog partial sums are per CTA of this size)

  // ------------------------------------------------------------------ validation (shared by the library and the host twin)
  inline int check_clover_lattice(const char *fn, const int X[4], int precision)
  {
    if (!X) return set_error(B200_ERR_INVALID, "%s: null argument", fn);
    for (int d = 0; d < 4; d++)
      if (X[d] <= 0 || (X[d] & 1)) return set_error(B200_ERR_INVALID, "%s: X[%d]=%d must be even and positive", fn, d, X[d]);
    if (precision != B200_DOUBLE && precision != B200_SINGLE)
      return set_error(B200_ERR_INVALID, "%s: precision %d not in {8,4}", fn, precision);
    return 0;
  }

  inline int check_compute_clover(const void *packed, const void *const qdp[4], const int X[4], const int border[4], int precision,
                                  double coeff)
  {
    const char *fn = "b200_compute_clover";
    if (!packed || !qdp || !border) return set_error(B200_ERR_INVALID, "%s: null argument", fn);
    for (int d = 0; d < 4; d++)
      if (!qdp[d]) return set_error(B200_ERR_INVALID, "%s: qdp[%d] is NULL", fn, d);
    if (int rc = check_clover_lattice(fn, X, precision)) return rc;
    for (int d = 0; d < 4; d++)
      if (border[d] != 0 && border[d] != 1) return set_error(B200_ERR_INVALID, "%s: border[%d]=%d not in {0,1}", fn, d, border[d]);
    if (!std::isfinite(coeff)) return set_error(B200_ERR_INVALID, "%s: coeff is not finite", fn);
    return 0;
  }

  inline int check_clover_invert(const double *trlog, const void *packed, const int X[4], int precision)
  {
    const char *fn = "b200_clover_invert_packed";
    if (!trlog || !packed) return set_error(B200_ERR_INVALID, "%s: null argument", fn);
    return check_clover_lattice(fn, X, precision);
  }

  // ------------------------------------------------------------------ site code: field strength -> A
  template <typename T> struct CloverBuildArgs {
    const T *u[4];
    T *out;
    int X[4], Xe[4], border[4];
    int volume_cb, volume_cb_e;
    T k; // coeff / 8: the 1/8 of F folded into the clover coefficient
  };

  template <typename T> void fill_clover_build(CloverBuildArgs<T> &a, const CloverBuildRequest &rq)
  {
    int V = 1, Ve = 1;
    for (int d = 0; d < 4; d++) {
      a.u[d] = reinterpret_cast<const T *>(rq.qdp[d]);
      a.X[d] = rq.X[d];
      a.border[d] = rq.border[d];
      a.Xe[d] = rq.X[d] + 2 * rq.border[d];
      V *= a.X[d];
      Ve *= a.Xe[d];
    }
    a.out = reinterpret_cast<T *>(rq.packed);
    a.volume_cb = V / 2;
    a.volume_cb_e = Ve / 2;
    a.k = (T)(rq.coeff * 0.125);
  }

  // U_mu at extended-lattice coordinates y + (dmu along mu) + (dnu along nu), wrapped periodically on the extended lattice
  // (border 0: the local block is periodic; border 1: the shift never leaves the halo)
  template <typename T>
  B2_HD void load_link_ext(T *u, const CloverBuildArgs<T> &a, int dir, const int *y, int mu, int dmu, int nu, int dnu)
  {
    int idx = 0, par = 0;
#pragma unroll
    for (int d = 3; d >= 0; d--) {
      const int z = y[d] + (d == mu ? dmu : 0) + (d == nu ? dnu : 0); // no runtime-indexed array: it would live in local memory
      const int c = z < 0 ? z + a.Xe[d] : (z >= a.Xe[d] ? z - a.Xe[d] : z);
      idx = idx * a.Xe[d] + c;
      par += c;
    }
    using V = std::conditional_t<sizeof(T) == 8, d2, f2>;
    const V *p = reinterpret_cast<const V *>(a.u[dir] + ((size_t)(par & 1) * a.volume_cb_e + (idx >> 1)) * 18);
#pragma unroll
    for (int i = 0; i < 9; i++) {
      const V w = ld<Cache::REUSE>(p + i);
      u[2 * i] = w.x;
      u[2 * i + 1] = w.y;
    }
  }

  // r = op(a) op(b) (acc: r += op(a) op(b)) for 3x3 complex matrices [3][3][2]; op = dagger where the flag is set
  template <bool da, bool db, bool acc = false, typename T> B2_HD void su3_mul_op(T *r, const T *a, const T *b)
  {
#pragma unroll
    for (int i = 0; i < 3; i++) {
#pragma unroll
      for (int j = 0; j < 3; j++) {
        T re = acc ? r[(i * 3 + j) * 2] : (T)0, im = acc ? r[(i * 3 + j) * 2 + 1] : (T)0;
#pragma unroll
        for (int k = 0; k < 3; k++) {
          const int ia = da ? (k * 3 + i) * 2 : (i * 3 + k) * 2, ib = db ? (j * 3 + k) * 2 : (k * 3 + j) * 2;
          const T ar = a[ia], ai = da ? -a[ia + 1] : a[ia + 1];
          const T br = b[ib], bi = db ? -b[ib + 1] : b[ib + 1];
          re = fma_rn(ar, br, re);
          re = fma_rn(-ai, bi, re);
          im = fma_rn(ar, bi, im);
          im = fma_rn(ai, br, im);
        }
        r[(i * 3 + j) * 2] = re;
        r[(i * 3 + j) * 2 + 1] = im;
      }
    }
  }

  // One link of a clover leaf: direction (0: mu, 1: nu), shifts along mu and nu, daggered or not
  struct LeafLink {
    int dir, dmu, dnu;
    bool dag;
  };
  // field_strength_tensor.cuh:57-157, each leaf U1 U2 U3 U4 in this order
  constexpr LeafLink kLeaf[4][4] = {
    {{0, 0, 0, false}, {1, 1, 0, false}, {0, 0, 1, true}, {1, 0, 0, true}},      // U_mu(x) U_nu(x+mu) U_mu(x+nu)^ U_nu(x)^
    {{1, 0, 0, false}, {0, -1, 1, true}, {1, -1, 0, true}, {0, -1, 0, false}},   // U_nu(x) U_mu(x+nu-mu)^ U_nu(x-mu)^ U_mu(x-mu)
    {{1, 0, -1, true}, {0, 0, -1, false}, {1, 1, -1, false}, {0, 0, 0, true}},   // U_nu(x-nu)^ U_mu(x-nu) U_nu(x+mu-nu) U_mu(x)^
    {{0, -1, 0, true}, {1, -1, -1, true}, {0, -1, -1, false}, {1, 0, -1, false}} // U_mu(x-mu)^ U_nu(x-mu-nu)^ U_mu(x-mu-nu) U_nu(x-nu)
  };

  template <int leaf, int l, typename T> B2_HD void leaf_link(T *u, const CloverBuildArgs<T> &a, const int *y, int mu, int nu)
  {
    constexpr LeafLink L = kLeaf[leaf][l];
    load_link_ext(u, a, L.dir ? nu : mu, y, mu, L.dmu, nu, L.dnu);
  }

  // q (+)= U1 U2 U3 U4 of one leaf (the first leaf sets q, the others add to it)
  template <int leaf, typename T> B2_HD void leaf_product(T *q, const CloverBuildArgs<T> &a, const int *y, int mu, int nu)
  {
    T u[18], v[18], w[18];
    leaf_link<leaf, 0>(u, a, y, mu, nu);
    leaf_link<leaf, 1>(v, a, y, mu, nu);
    su3_mul_op<kLeaf[leaf][0].dag, kLeaf[leaf][1].dag>(w, u, v);
    leaf_link<leaf, 2>(u, a, y, mu, nu);
    su3_mul_op<false, kLeaf[leaf][2].dag>(v, w, u);
    leaf_link<leaf, 3>(u, a, y, mu, nu);
    su3_mul_op<false, kLeaf[leaf][3].dag, leaf != 0>(q, v, u);
  }

  // The chiral blocks need, per chirality, S1 = F10 -+ F32 (imaginary diagonal and strictly-lower entries: 9 reals) and
  // S2 = F20 +- F31 - i (F21 -+ F30) (18 reals), both without the 1/8.  Weight w of a plane's G = Q - Q^dagger in them:
  // 0: +1, 1: -1, 2: +i, 3: -i.
  template <typename T> B2_HD void add_weighted(T &re, T &im, T gr, T gi, int w)
  {
    const T tr = w < 2 ? gr : -gi, ti = w < 2 ? gi : gr;
    if (w & 1) {
      re -= tr;
      im -= ti;
    } else {
      re += tr;
      im += ti;
    }
  }

  // plane p: (mu, nu), target (0: S1, 1: S2), weight in chirality 0 and 1 (clover_compute.cuh:82-85)
  struct PlaneMap {
    int mu, nu, s2, w0, w1;
  };
  B2_HD PlaneMap plane_map(int p)
  {
    switch (p) {
    case 0: return {1, 0, 0, 0, 0}; // F10: S1 += G, S1 += G
    case 1: return {2, 0, 1, 0, 0}; // F20: S2 += G, S2 += G
    case 2: return {2, 1, 1, 3, 3}; // F21: S2 -= i G, S2 -= i G
    case 3: return {3, 0, 1, 2, 3}; // F30: S2 += i G, S2 -= i G
    case 4: return {3, 1, 1, 0, 1}; // F31: S2 += G, S2 -= G
    default: return {3, 2, 0, 1, 0}; // F32: S1 -= G, S1 += G
    }
  }

  template <typename T> B2_HD void add_plane(T (&s1)[2][9], T (&s2)[2][18], const CloverBuildArgs<T> &a, const int *y, int p)
  {
    const PlaneMap m = plane_map(p);
    T q[18];
#pragma unroll 1
    for (int leaf = 0; leaf < 4; leaf++) { // one leaf's loads at a time, as for the planes
      switch (leaf) {
      case 0: leaf_product<0>(q, a, y, m.mu, m.nu); break;
      case 1: leaf_product<1>(q, a, y, m.mu, m.nu); break;
      case 2: leaf_product<2>(q, a, y, m.mu, m.nu); break;
      default: leaf_product<3>(q, a, y, m.mu, m.nu); break;
      }
    }
    // G = Q - Q^dagger: G(i,j) = (Q(i,j).re - Q(j,i).re, Q(i,j).im + Q(j,i).im)
    auto g = [&](int i, int j, T &gr, T &gi) {
      gr = q[(i * 3 + j) * 2] - q[(j * 3 + i) * 2];
      gi = q[(i * 3 + j) * 2 + 1] + q[(j * 3 + i) * 2 + 1];
    };
    if (!m.s2) {
      constexpr int lo[3][2] = {{1, 0}, {2, 0}, {2, 1}};
#pragma unroll
      for (int i = 0; i < 3; i++) {
        T gr, gi; // S1 weights are +-1: the imaginary diagonal is weight * Im G(i,i)
        g(i, i, gr, gi);
        s1[0][i] += m.w0 ? -gi : gi;
        s1[1][i] += m.w1 ? -gi : gi;
        g(lo[i][0], lo[i][1], gr, gi);
        add_weighted(s1[0][3 + 2 * i], s1[0][4 + 2 * i], gr, gi, m.w0);
        add_weighted(s1[1][3 + 2 * i], s1[1][4 + 2 * i], gr, gi, m.w1);
      }
    } else {
#pragma unroll
      for (int i = 0; i < 3; i++) {
#pragma unroll
        for (int j = 0; j < 3; j++) {
          T gr, gi;
          g(i, j, gr, gi);
          add_weighted(s2[0][(i * 3 + j) * 2], s2[0][(i * 3 + j) * 2 + 1], gr, gi, m.w0);
          add_weighted(s2[1][(i * 3 + j) * 2], s2[1][(i * 3 + j) * 2 + 1], gr, gi, m.w1);
        }
      }
    }
  }

  // A at local site (x_cb, parity): both chiral blocks, 72 reals at out[(parity Vh + x_cb) 72]
  template <typename T> B2_HD void clover_build_site(const CloverBuildArgs<T> &a, int x_cb, int parity)
  {
    Geom g;
    geom_init(g, a.X);
    int y[4];
    coords_from_cb(y, g, x_cb, parity);
    for (int d = 0; d < 4; d++) y[d] += a.border[d];
    T s1[2][9], s2[2][18];
#pragma unroll
    for (int c = 0; c < 2; c++) {
#pragma unroll
      for (int i = 0; i < 9; i++) s1[c][i] = 0;
#pragma unroll
      for (int i = 0; i < 18; i++) s2[c][i] = 0;
    }
    // one plane at a time (not unrolled): the compiler would otherwise hoist the link loads of several planes and spill
#pragma unroll 1
    for (int p = 0; p < 6; p++) add_plane(s1, s2, a, y, p);
    T *out = a.out + ((size_t)parity * a.volume_cb + x_cb) * 72;
    const T k = a.k;
#pragma unroll
    for (int c = 0; c < 2; c++) {
      T *o = out + 36 * c;
      // A = 1 - (i k S1) on the upper 3x3, 1 + (i k S1) on the lower one, k S2 in the off-diagonal 3x3
#pragma unroll
      for (int i = 0; i < 3; i++) {
        const T d = mul_rn(k, s1[c][i]);
        o[i] = (T)1 + d;
        o[i + 3] = (T)1 - d;
      }
      constexpr int lo[3][2] = {{1, 0}, {2, 0}, {2, 1}};
#pragma unroll
      for (int n = 0; n < 3; n++) {
        const T k_re = mul_rn(k, s1[c][3 + 2 * n]), k_im = mul_rn(k, s1[c][4 + 2 * n]);
        const int u = tri_idx(lo[n][0], lo[n][1]), l = tri_idx(lo[n][0] + 3, lo[n][1] + 3);
        o[u] = k_im; // -i k S1(i,j)
        o[u + 1] = -k_re;
        o[l] = -k_im; // +i k S1(i,j)
        o[l + 1] = k_re;
      }
#pragma unroll
      for (int i = 0; i < 3; i++) {
#pragma unroll
        for (int j = 0; j < 3; j++) {
          const int t = tri_idx(i + 3, j);
          o[t] = mul_rn(k, s2[c][(i * 3 + j) * 2]);
          o[t + 1] = mul_rn(k, s2[c][(i * 3 + j) * 2 + 1]);
        }
      }
    }
  }

  // ------------------------------------------------------------------ site code: Cholesky -> A^-1, log det A
  // One 6x6 block a (packed order) -> inv (packed order, nullptr: none); returns log det = 2 sum_j log L_jj.
  // A = L L^dagger in double whatever T is (clover_field.h:52-75: CLOVER_PROMOTE_CHOLESKY); A^-1 = M^dagger M, M = L^-1.
  template <typename T> B2_HD double clover_block_invert(T *inv, const T *a)
  {
    double Lr[6][6], Li[6][6], d[6], rd[6];
    double logdet = 0.0;
#pragma unroll
    for (int j = 0; j < 6; j++) {
      double s = (double)a[j];
#pragma unroll
      for (int k = 0; k < 6; k++) {
        if (k >= j) continue;
        s = fma_rn(-Lr[j][k], Lr[j][k], s);
        s = fma_rn(-Li[j][k], Li[j][k], s);
      }
      d[j] = std::sqrt(s);
      rd[j] = 1.0 / d[j];
      logdet += 2.0 * std::log(d[j]);
#pragma unroll
      for (int i = 0; i < 6; i++) {
        if (i <= j) continue;
        const int t = tri_idx(i, j);
        double re = (double)a[t], im = (double)a[t + 1];
#pragma unroll
        for (int k = 0; k < 6; k++) { // - L(i,k) conj(L(j,k))
          if (k >= j) continue;
          re = fma_rn(-Lr[i][k], Lr[j][k], re);
          re = fma_rn(-Li[i][k], Li[j][k], re);
          im = fma_rn(-Li[i][k], Lr[j][k], im);
          im = fma_rn(Lr[i][k], Li[j][k], im);
        }
        Lr[i][j] = mul_rn(re, rd[j]);
        Li[i][j] = mul_rn(im, rd[j]);
      }
    }
    if (!inv) return logdet;
    // M = L^-1 (lower): M(j,j) = 1 / L(j,j); M(i,j) = -(sum_{j<=k<i} L(i,k) M(k,j)) / L(i,i)
    double Mr[6][6], Mi[6][6];
#pragma unroll
    for (int j = 0; j < 6; j++) {
      Mr[j][j] = rd[j];
      Mi[j][j] = 0.0;
#pragma unroll
      for (int i = 0; i < 6; i++) {
        if (i <= j) continue;
        double re = 0.0, im = 0.0;
#pragma unroll
        for (int k = 0; k < 6; k++) {
          if (k < j || k >= i) continue;
          re = fma_rn(Lr[i][k], Mr[k][j], re);
          re = fma_rn(-Li[i][k], Mi[k][j], re);
          im = fma_rn(Lr[i][k], Mi[k][j], im);
          im = fma_rn(Li[i][k], Mr[k][j], im);
        }
        Mr[i][j] = -mul_rn(re, rd[i]);
        Mi[i][j] = -mul_rn(im, rd[i]);
      }
    }
    // A^-1(i,j) = sum_{k >= i} conj(M(k,i)) M(k,j) for i >= j
#pragma unroll
    for (int i = 0; i < 6; i++) {
#pragma unroll
      for (int j = 0; j < 6; j++) {
        if (j > i) continue;
        double re = 0.0, im = 0.0;
#pragma unroll
        for (int k = 0; k < 6; k++) {
          if (k < i) continue;
          re = fma_rn(Mr[k][i], Mr[k][j], re);
          re = fma_rn(Mi[k][i], Mi[k][j], re);
          im = fma_rn(Mr[k][i], Mi[k][j], im);
          im = fma_rn(-Mi[k][i], Mr[k][j], im);
        }
        if (i == j) {
          inv[i] = (T)re;
        } else {
          const int t = tri_idx(i, j);
          inv[t] = (T)re;
          inv[t + 1] = (T)im;
        }
      }
    }
    return logdet;
  }

  // both chiral blocks of packed site `site` (= parity Vh + x_cb); returns their summed log det
  template <typename T> B2_HD double clover_invert_site(T *inv, const T *packed, size_t site)
  {
    double s = 0.0;
#pragma unroll
    for (int c = 0; c < 2; c++) s += clover_block_invert<T>(inv ? inv + site * 72 + 36 * c : nullptr, packed + site * 72 + 36 * c);
    return s;
  }

  // Fixed-order tree over kCloverBuildThreads values (what one CTA does in shared memory between barriers)
  B2_HD void clover_tree_step(double *s, int tid, int w)
  {
    if (tid < w) s[tid] += s[tid + w];
  }

  // ------------------------------------------------------------------ entry points (executor E: the CUDA library or the twin)
  template <typename T> int launch_clover_build(const CloverBuildRequest &rq);   // inst_clover_build.cu
  template <typename T> int launch_clover_invert(const CloverInvertRequest &rq); // inst_clover_build.cu

  template <class E>
  int compute_clover(void *packed, const void *const qdp[4], const int X[4], const int border[4], int precision, double coeff, void *stream)
  {
    if (int rc = check_compute_clover(packed, qdp, X, border, precision, coeff)) return rc;
    if (int rc = E::require_device()) return rc;
    CloverBuildRequest rq;
    for (int d = 0; d < 4; d++) {
      rq.qdp[d] = qdp[d];
      rq.X[d] = X[d];
      rq.border[d] = border[d];
    }
    rq.packed = packed;
    rq.coeff = coeff;
    rq.stream = stream;
    return precision == B200_DOUBLE ? E::template clover_build<double>(rq) : E::template clover_build<float>(rq);
  }

  template <class E> int clover_invert_packed(void *inv, double trlog[2], const void *packed, const int X[4], int precision, void *stream)
  {
    if (int rc = check_clover_invert(trlog, packed, X, precision)) return rc;
    if (int rc = E::require_device()) return rc;
    CloverInvertRequest rq;
    for (int d = 0; d < 4; d++) rq.X[d] = X[d];
    rq.inv = inv;
    rq.packed = packed;
    rq.trlog = trlog;
    rq.stream = stream;
    return precision == B200_DOUBLE ? E::template clover_invert<double>(rq) : E::template clover_invert<float>(rq);
  }

} // namespace b200
