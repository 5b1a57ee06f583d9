// C entry points of the operator / solver layer (declared in include/b200_dslash.h).
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "dirac.h"

namespace b200
{
  int set_error(int code, const char *fmt, ...);
  int require_device();
}

using namespace b200::host;

struct b200_dirac_s {
  GaugeField U;
  CloverField A;
  bool has_clover = false;
  CommContext comm;
  bool has_comm = false;
  b200_comm *user_comm = nullptr; // the caller's exchange: pull_comm mirrors it into `comm` before every call
  int precision = 0;
  int X[4];
  std::unique_ptr<Dirac> op;
};

// Mirror the caller's b200_comm into the operator's CommContext.  The exchange / reduction sequence numbers are NOT
// copied: every operator created on one b200_comm advances the caller's counters through these pointers, so a precise
// and a sloppy operator sharing an exchange (or Python code using the same HaloExchange) can never reuse a sequence
// number or disagree on the buffer parity.
static void pull_comm(b200_dirac_s *h)
{
  if (!h->has_comm) return;
  b200_comm *c = h->user_comm;
  CommContext &k = h->comm;
  memcpy(k.comm_dim, c->comm_dim, sizeof(k.comm_dim));
  memcpy(k.send_dst, c->send_dst, sizeof(k.send_dst));
  memcpy(k.send_signal, c->send_signal, sizeof(k.send_signal));
  memcpy(k.recv, c->recv, sizeof(k.recv));
  memcpy(k.recv_flag, c->recv_flag, sizeof(k.recv_flag));
  k.block_counter = c->block_counter;
  k.timeout_flag = c->timeout_flag;
  k.seq_shared = &c->seq;
  k.pack_stream = c->pack_stream;
  k.allreduce_sum = c->allreduce_sum;
  k.user = c->user;
  k.rank = c->rank;
  k.n_ranks = c->n_ranks;
  memcpy(k.reduce_peer, c->reduce_peer, sizeof(k.reduce_peer));
  k.reduce_seq_shared = &c->reduce_seq;
}

template <typename F> static int guarded(F &&f)
{
  try {
    f();
    return B200_SUCCESS;
  } catch (const Error &e) {
    return b200::set_error(B200_ERR_INVALID, "%s", e.what());
  } catch (const std::exception &e) {
    return b200::set_error(B200_ERR_INVALID, "unexpected: %s", e.what());
  }
}

static ColorSpinorField wrap(const b200_dirac_s *h, const b200_spinor *s)
{
  if (!s || !s->v) throw Error("null spinor");
  return ColorSpinorField::wrap(s->v, h->X, h->precision, s->n_parity);
}

extern "C" {

int b200_dirac_create(b200_dirac **out, int type, int precision, const int X[4], const b200_gauge *U, const b200_clover *A,
                      const b200_clover *Ainv, double kappa, int matpc_type, b200_comm *comm, void *stream)
{
  return guarded([&] {
    if (!out || !U || !X) throw Error("b200_dirac_create: null argument");
    auto h = std::make_unique<b200_dirac_s>();
    h->precision = precision;
    h->U.g = *U;
    h->U.precision = precision;
    for (int d = 0; d < 4; d++) h->X[d] = h->U.X[d] = X[d];
    if (A) {
      h->A.c = *A;
      if (Ainv) h->A.cinv = *Ainv;
      h->A.precision = precision;
      h->has_clover = true;
    }
    if (comm) {
      h->has_comm = true;
      h->user_comm = comm;
      pull_comm(h.get());
    }
    DiracParam p;
    p.gauge = &h->U;
    p.clover = h->has_clover ? &h->A : nullptr;
    p.kappa = kappa;
    p.matpcType = (QudaMatPCType)matpc_type;
    p.comm = h->has_comm ? &h->comm : nullptr;
    p.stream = stream;
    static const char *names[] = {"wilson", "wilsonpc", "clover", "cloverpc", "twistedmass", "twistedmasspc"};
    if (type < 0 || type > 5) throw Error("b200_dirac_create: unknown operator type");
    h->op.reset(Dirac::create(names[type], p));
    *out = h.release();
  });
}

int b200_dirac_set_twist(b200_dirac *op, double mu)
{
  return guarded([&] {
    if (!op) throw Error("b200_dirac_set_twist: null operator");
    if (!op->op->is_twisted()) throw Error("b200_dirac_set_twist: not a twisted-mass operator");
    op->op->setMu(mu);
  });
}

int b200_dirac_destroy(b200_dirac *op)
{
  delete op;
  return B200_SUCCESS;
}

int b200_dirac_apply(b200_dirac *h, int what, const b200_spinor *out, const b200_spinor *in, int parity,
                     const b200_spinor *x, double k, int dagger)
{
  return guarded([&] {
    if (!h) throw Error("null operator");
    pull_comm(h);
    auto o = wrap(h, out), i = wrap(h, in);
    if (dagger) h->op->flipDagger();
    try {
      switch (what) {
      case B200_APPLY_M: h->op->M(o, i); break;
      case B200_APPLY_MDAG: h->op->Mdag(o, i); break;
      case B200_APPLY_MDAGM: h->op->MdagM(o, i); break;
      case B200_APPLY_DSLASH: h->op->Dslash(o, i, parity); break;
      case B200_APPLY_DSLASH_XPAY: {
        auto xf = wrap(h, x);
        h->op->DslashXpay(o, i, parity, xf, k);
      } break;
      default: throw Error("b200_dirac_apply: unknown operation");
      }
    } catch (...) {
      if (dagger) h->op->flipDagger();
      throw;
    }
    if (dagger) h->op->flipDagger();
  });
}

/* 0 if no halo wait has given up since the last check on this exchange; B200_ERR_CUDA (and the flag is cleared) otherwise.
 * Synchronises `stream`.  The solvers check by themselves; callers of b200_dirac_apply / b200_dslash_apply on partitioned
 * lattices call this at their own synchronisation points. */
int b200_comm_check(b200_comm *c, void *stream)
{
  return guarded([&] {
    if (!c) throw Error("b200_comm_check: null exchange");
    CommContext k;
    k.timeout_flag = c->timeout_flag;
    if (halo_timed_out(&k, stream)) throw Error("a halo wait timed out (a neighbour's faces never arrived): results since the last check are not valid");
  });
}

int b200_dirac_prepare(b200_dirac *h, const b200_spinor *x, const b200_spinor *b, int *src_parity, int *sol_parity)
{
  return guarded([&] {
    pull_comm(h);
    auto xf = wrap(h, x), bf = wrap(h, b);
    ColorSpinorField sol, src;
    h->op->prepare(sol, src, xf, bf, QUDA_MAT_SOLUTION);
    const size_t pb = xf.parity_bytes;
    if (src_parity) *src_parity = (int)((static_cast<char *>(src.v) - static_cast<char *>(xf.v)) / (long)pb);
    if (sol_parity) *sol_parity = (int)((static_cast<char *>(sol.v) - static_cast<char *>(xf.v)) / (long)pb);
  });
}

int b200_dirac_reconstruct(b200_dirac *h, const b200_spinor *x, const b200_spinor *b)
{
  return guarded([&] {
    pull_comm(h);
    auto xf = wrap(h, x), bf = wrap(h, b);
    h->op->reconstruct(xf, bf, QUDA_MAT_SOLUTION);
  });
}

} // extern "C"

using Solver = void (*)(const Dirac &, const Dirac &, ColorSpinorField &, const ColorSpinorField &, SolverParam &);

// argument checks and comm mirroring shared by the solver entry points: `check` refuses a bad parameter block before a
// device is needed, `solve(precise, sloppy)` runs the solve
template <typename C, typename F>
static int invert(const char *name, b200_dirac *precise, b200_dirac *sloppy, const void *param, C &&check, F &&solve)
{
  if (!precise || !param) return b200::set_error(B200_ERR_INVALID, "%s: null argument", name);
  try {
    check();
  } catch (const Error &e) {
    return b200::set_error(B200_ERR_INVALID, "%s: %s", name, e.what());
  }
  if (int rc = b200::require_device()) return rc;
  return guarded([&] {
    if (!sloppy) sloppy = precise;
    pull_comm(precise);
    if (sloppy != precise) {
      // a partitioned mixed-precision solve needs one halo context per precision (the ghost buffers differ in size);
      // both advance in lock step on every rank because all ranks execute the same operator sequence
      if (precise->has_comm != sloppy->has_comm) throw Error("precise / sloppy operators disagree on partitioning");
      pull_comm(sloppy);
    }
    solve(*precise, *sloppy);
  });
}

// parameter marshaling of the single-system solvers
static int invert(const char *name, Solver solve, b200_dirac *precise, b200_dirac *sloppy, const b200_spinor *x,
                  const b200_spinor *b, b200_solver_param *param)
{
  return invert(name, precise, sloppy, param, [] {}, [&](b200_dirac_s &pr, b200_dirac_s &sl) {
    auto xf = wrap(&pr, x), bf = wrap(&pr, b);
    SolverParam sp;
    sp.tol = param->tol;
    sp.maxiter = param->maxiter;
    sp.delta = param->delta > 0 ? param->delta : 0.1;
    solve(*pr.op, *sl.op, xf, bf, sp);
    param->iter = sp.iter;
    param->reliable_updates = sp.reliable_updates;
    param->true_res = sp.true_res;
    param->secs = sp.secs;
    param->gflops = sp.gflops;
    param->host_syncs = sp.host_syncs;
  });
}

extern "C" {

int b200_invert_bicgstab(b200_dirac *precise, b200_dirac *sloppy, const b200_spinor *x, const b200_spinor *b, b200_solver_param *param)
{
  return invert("b200_invert_bicgstab", invertBiCGStab, precise, sloppy, x, b, param);
}

int b200_invert_cg(b200_dirac *precise, b200_dirac *sloppy, const b200_spinor *x, const b200_spinor *b, b200_solver_param *param)
{
  return invert("b200_invert_cg", invertCG, precise, sloppy, x, b, param);
}

int b200_invert_multishift_cg(b200_dirac *precise, b200_dirac *sloppy, const b200_spinor *x, const b200_spinor *b,
                              b200_multishift_param *param)
{
  MultiShiftParam mp;
  auto check = [&] {
    mp.n_shift = param->n_shift;
    memcpy(mp.offset, param->offset, sizeof(mp.offset));
    memcpy(mp.tol_offset, param->tol_offset, sizeof(mp.tol_offset));
    mp.maxiter = param->maxiter;
    mp.delta = param->delta > 0 ? param->delta : 0.1;
    checkMultiShiftParam(mp);
    if (!x || !b) throw Error("null spinor");
    for (int j = 0; j < mp.n_shift; j++)
      if (!x[j].v) throw Error("solution descriptor " + std::to_string(j) + " has no field");
  };
  return invert("b200_invert_multishift_cg", precise, sloppy, param, check, [&](b200_dirac_s &pr, b200_dirac_s &sl) {
    std::vector<ColorSpinorField> xs;
    for (int j = 0; j < mp.n_shift; j++) xs.push_back(wrap(&pr, &x[j]));
    auto bf = wrap(&pr, b);
    invertMultiShiftCG(*pr.op, *sl.op, xs, bf, mp);
    param->iter = mp.iter;
    for (int j = 0; j < B200_MAX_SHIFTS; j++) {
      const bool on = j < mp.n_shift;
      param->iter_offset[j] = on ? mp.iter_offset[j] : 0;
      param->refine_iter[j] = on ? mp.refine_iter[j] : 0;
      param->iter_res_offset[j] = on ? mp.iter_res_offset[j] : 0.0;
      param->true_res_offset[j] = on ? mp.true_res_offset[j] : 0.0;
    }
    param->reliable_updates = mp.reliable_updates;
    param->secs = mp.secs;
    param->gflops = mp.gflops;
    param->host_syncs = mp.host_syncs;
  });
}

int b200_clover_force(void *mom, double dt, const b200_spinor *x, const double *coeff, double kappa2, double ck, int n,
                      double multiplicity, const void *const qdp[4], const void *packed, b200_dirac *op)
{
  const char *name = "b200_clover_force";
  if (!mom || !x || !coeff || !qdp || !packed || !op) return b200::set_error(B200_ERR_INVALID, "%s: null argument", name);
  if (n < 1 || n > B200_MAX_SHIFTS) return b200::set_error(B200_ERR_INVALID, "%s: n=%d not in [1, %d]", name, n, B200_MAX_SHIFTS);
  const Dirac &d = *op->op;
  if (!d.is_clover() || !d.pc() || d.is_symmetric() || (op->has_comm && op->user_comm && [&] {
        pull_comm(op);
        return op->comm.partitioned();
      }()))
    return b200::set_error(B200_ERR_INVALID, "%s: needs an asymmetric \"cloverpc\" operator on an unpartitioned lattice", name);
  if (int rc = b200::require_device()) return rc;
  return guarded([&] {
    std::vector<ColorSpinorField> xs;
    for (int i = 0; i < n; i++) xs.push_back(wrap(op, &x[i]));
    computeCloverForce(mom, dt, xs, coeff, kappa2, ck, multiplicity, qdp, packed, d);
  });
}
}
