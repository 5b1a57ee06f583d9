// Host-side C++ layer above the C ABI for the Wilson / Wilson-clover / twisted-mass family: what a QUDA caller reaches
// through Dirac::M / MdagM / prepare / reconstruct and invertQuda's CG and BiCGStab.
//   reference surface   include/dslash_quda.h:83-811 (Apply*), include/dirac_quda.h (Dirac* classes),
//                       lib/blas_quda.cu + lib/reduce_quda.cu (blas), lib/inv_cg_quda.cpp:63-420 (CG, reliable updates),
//                       lib/inv_bicgstab_quda.cpp (BiCGStab), lib/inv_multi_cg_quda.cpp (multi-shift CG)
// Design (not a mirror of the reference's class tree):
//   * ONE operator class.  An even-odd operator is described by its site term A (identity, clover, twist) and whether it
//     is the full matrix or the Schur complement; M / Mdag / prepare / reconstruct are short sequences of two
//     primitives -- `hop` (a Dslash launch with the site term fused into its epilogue) and `site` (A or A^-1 alone).
//   * Everything runs on the operator's stream: Dslash, blas, reductions, the NVLink all-reduce.  Reductions are
//     two-stage and summed in a fixed order (bit-reproducible); their results stay on the device -- each solver's
//     scalars (CG's alpha, beta; BiCGStab's rho, alpha, omega, beta; multi-shift CG's per-shift zeta, alpha, beta) are
//     computed there and consumed by the next kernel,
//     the host only follows one iteration behind to decide convergence / reliable updates, so no iteration waits for a
//     host round trip.
// Errors throw b200::host::Error (the analogue of errorQuda); everything bottoms out in include/b200_dslash.h.
#pragma once

#include <array>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../../include/b200_dslash.h"

namespace b200
{
  namespace host
  {

    struct Error : std::runtime_error {
      using std::runtime_error::runtime_error;
    };

    enum QudaParity { QUDA_EVEN_PARITY = 0, QUDA_ODD_PARITY = 1, QUDA_INVALID_PARITY = -1 };
    enum QudaMatPCType {
      QUDA_MATPC_EVEN_EVEN = 0,
      QUDA_MATPC_ODD_ODD = 1,
      QUDA_MATPC_EVEN_EVEN_ASYMMETRIC = 2,
      QUDA_MATPC_ODD_ODD_ASYMMETRIC = 3
    };
    enum QudaSolutionType { QUDA_MAT_SOLUTION, QUDA_MATPC_SOLUTION, QUDA_MATPCDAG_MATPC_SOLUTION };

    // Halo context handed in by whoever bootstrapped the ranks (quda_b200/comm.py over torch.distributed):
    // peer-mapped ghost slabs of the neighbours, local flags, and an allreduce callback for the solver's scalars.
    struct CommContext {
      int comm_dim[4] = {0, 0, 0, 0};
      // [buffer][dim][face]: where our faces go (peer memory) and the flag to raise there
      void *send_dst[2][4][2] = {};
      void *send_signal[2][4][2] = {};
      // [buffer][dim][dir]: local receive buffers and the flags the neighbours raise
      void *recv[2][4][2] = {};
      void *recv_flag[2][4][2] = {};
      int *block_counter = nullptr;
      int *timeout_flag = nullptr;
      unsigned *seq_shared = nullptr; // the ONE exchange counter all operators on this exchange advance (b200_comm::seq)
      unsigned seq_local = 0;         // used when seq_shared is null
      void *pack_stream = nullptr; // cudaStream_t for the pack kernels (nullptr: same stream as the Dslash)
      void (*allreduce_sum)(double *data, int n, void *user) = nullptr; // nullptr: single rank
      void *user = nullptr;
      // NVLink mailbox all-reduce (b200_comm::reduce_peer); n_ranks == 0: use the callback
      int rank = 0, n_ranks = 0;
      void *reduce_peer[B200_MAX_RANKS] = {};
      unsigned *reduce_seq_shared = nullptr;
      unsigned reduce_seq_local = 0;
      bool partitioned() const { return comm_dim[0] || comm_dim[1] || comm_dim[2] || comm_dim[3]; }
      unsigned &seq() { return seq_shared ? *seq_shared : seq_local; }
      unsigned &reduce_seq() { return reduce_seq_shared ? *reduce_seq_shared : reduce_seq_local; }
      bool mailboxes() const { return n_ranks >= 2 && reduce_peer[0] != nullptr; }
    };

    class ColorSpinorField
    {
      std::shared_ptr<void> owned;

    public:
      void *v = nullptr;
      int X[4] = {0, 0, 0, 0};
      int precision = 0; // bytes per real: 8, 4, 2
      int n_parity = 1;
      size_t parity_bytes = 0; // bytes of one parity block (data + norms)

      static ColorSpinorField create(const int *X, int precision, int n_parity);
      static ColorSpinorField wrap(void *v, const int *X, int precision, int n_parity);
      int VolumeCB() const { return X[0] * X[1] * X[2] * X[3] / 2; }
      size_t Bytes() const { return parity_bytes * n_parity; }
      size_t Length() const { return (size_t)24 * VolumeCB() * n_parity; } // reals
      template <typename T> T *data() const { return static_cast<T *>(v); }   // v as reals of type T
      ColorSpinorField parity_view(int p) const; // Even()/Odd() of a full field
      ColorSpinorField Even() const { return parity_view(0); }
      ColorSpinorField Odd() const { return parity_view(1); }
      b200_spinor desc() const;
    };

    struct GaugeField {
      b200_gauge g {};
      int X[4] = {0, 0, 0, 0};
      int precision = 0;
    };

    struct CloverField {
      b200_clover c {};     // the direct term A (and the only field for dynamic-inverse builds)
      b200_clover cinv {};  // A^{-1} for static inversion (clover pointer may be null when dynamic)
      int precision = 0;
      bool has_inverse() const { return cinv.clover != nullptr; }
    };

    // ---- the drop-in entry points (reference: include/dslash_quda.h); on a partitioned lattice they own the halo
    // exchange exactly as the reference's do (pack + remote write on the side stream, interior, boundary)
    void ApplyWilson(ColorSpinorField &out, const ColorSpinorField &in, const GaugeField &U, double a,
                     const ColorSpinorField &x, int parity, bool dagger, const int *comm_override, CommContext *comm,
                     void *stream = nullptr);
    void ApplyWilsonClover(ColorSpinorField &out, const ColorSpinorField &in, const GaugeField &U, const CloverField &A,
                           double a, const ColorSpinorField &x, int parity, bool dagger, const int *comm_override,
                           CommContext *comm, void *stream = nullptr);
    void ApplyWilsonCloverPreconditioned(ColorSpinorField &out, const ColorSpinorField &in, const GaugeField &U,
                                         const CloverField &A, double a, const ColorSpinorField &x, int parity,
                                         bool dagger, const int *comm_override, CommContext *comm, void *stream = nullptr);
    void ApplyClover(ColorSpinorField &out, const ColorSpinorField &in, const CloverField &A, bool inverse, int parity,
                     void *stream = nullptr);
    // degenerate twisted mass (include/dslash_quda.h:363-406,883)
    void ApplyTwistedMass(ColorSpinorField &out, const ColorSpinorField &in, const GaugeField &U, double a, double b,
                          const ColorSpinorField &x, int parity, bool dagger, const int *comm_override, CommContext *comm,
                          void *stream = nullptr);
    void ApplyTwistedMassPreconditioned(ColorSpinorField &out, const ColorSpinorField &in, const GaugeField &U, double a,
                                        double b, bool xpay, const ColorSpinorField &x, int parity, bool dagger,
                                        bool asymmetric, const int *comm_override, CommContext *comm, void *stream = nullptr);
    void ApplyTwistGamma(ColorSpinorField &out, const ColorSpinorField &in, double kappa, double mu, bool dagger, bool inverse,
                         void *stream = nullptr);

    // where blas kernels and reductions run: the operator's stream and (for global sums) its halo context
    struct Exec {
      void *stream = nullptr;
      CommContext *comm = nullptr;
    };

    // ---- blas on native-order fields (fp64 / fp32); reductions accumulate in double, in a fixed order
    namespace blas
    {
      void copy(ColorSpinorField &dst, const ColorSpinorField &src, const Exec &ex); // precision conversion allowed (8 <-> 4)
      void zero(ColorSpinorField &x, const Exec &ex);
      void axpy(double a, const ColorSpinorField &x, ColorSpinorField &y, const Exec &ex); // y += a x
      // the reductions below synchronise the stream (they return the global sum to the host)
      double norm2(const ColorSpinorField &x, const Exec &ex);
      double axpyNorm(double a, const ColorSpinorField &x, ColorSpinorField &y, const Exec &ex); // y += a x ; |y|^2
      long long flops();
    } // namespace blas

    struct DiracParam {
      const GaugeField *gauge = nullptr;
      const CloverField *clover = nullptr;
      double kappa = 0.0;
      double mu = 0.0; // twisted mass
      QudaMatPCType matpcType = QUDA_MATPC_EVEN_EVEN;
      bool dagger = false;
      int commDim[4] = {1, 1, 1, 1};
      CommContext *comm = nullptr;
      void *stream = nullptr;
    };

    // site term of the even-odd operator  M = [[A_e, -kappa D_eo], [-kappa D_oe, A_o]]
    enum class SiteTerm { Identity, Clover, Twist };

    class Dirac
    {
      const GaugeField *gauge;
      const CloverField *clover;
      double kappa, mu;
      QudaMatPCType matpcType;
      mutable bool dagger;
      int commDim[4];
      CommContext *comm;
      void *stream;
      SiteTerm term;
      bool schur;           // operator acts on one parity (Schur complement of the even-odd decomposition)
      bool symmetric;       // Schur form 1 - k^2 A^-1 D A^-1 D (else A - k^2 D A^-1 D)
      int this_parity, other_parity;
      mutable long long dslash_applications = 0;

      // primitives
      enum class Fuse { None, A, AinvPost }; // what the Dslash epilogue applies: nothing / A on x / A^-1 on D in
      void hop(ColorSpinorField &out, const ColorSpinorField &in, int parity, Fuse f, const ColorSpinorField *x, double k) const;
      void site(ColorSpinorField &out, const ColorSpinorField &in, int parity, bool inverse) const;

    public:
      Dirac(SiteTerm term, bool schur, const DiracParam &p);
      // "wilson", "wilsonpc", "clover", "cloverpc", "twistedmass", "twistedmasspc"
      static Dirac *create(const std::string &type, const DiracParam &p);

      void Dslash(ColorSpinorField &out, const ColorSpinorField &in, int parity) const;
      void DslashXpay(ColorSpinorField &out, const ColorSpinorField &in, int parity, const ColorSpinorField &x, double k) const;
      void M(ColorSpinorField &out, const ColorSpinorField &in) const;
      void Mdag(ColorSpinorField &out, const ColorSpinorField &in) const;
      void MdagM(ColorSpinorField &out, const ColorSpinorField &in) const;
      void prepare(ColorSpinorField &sol, ColorSpinorField &src, ColorSpinorField &x, const ColorSpinorField &b, QudaSolutionType) const;
      void reconstruct(ColorSpinorField &x, const ColorSpinorField &b, QudaSolutionType) const;

      bool pc() const { return schur; }
      bool is_twisted() const { return term == SiteTerm::Twist; }
      void setMu(double m) { mu = m; }
      void setCommDim(const int *c) { for (int d = 0; d < 4; d++) commDim[d] = c[d]; }
      void flipDagger() const { dagger = !dagger; }
      long long DslashApplications() const { return dslash_applications; }
      CommContext *Comm() const { return comm; }
      void *Stream() const { return stream; }
      int Precision() const { return gauge->precision; }
      Exec exec() const { return Exec {stream, comm}; }
    };

    // ---- CG on MdagM with optional mixed precision + reliable updates (behaviour of lib/inv_cg_quda.cpp:63-420)
    struct SolverParam {
      double tol = 1e-10;
      int maxiter = 10000;
      double delta = 0.1;       // reliable-update threshold (QudaInvertParam::reliable_delta)
      // results
      int iter = 0;
      double true_res = 0.0;
      double secs = 0.0;
      double gflops = 0.0;
      int reliable_updates = 0;
      int host_syncs = 0; // stream synchronisations the solve needed (diagnostic: ~1 per iteration, off the critical path)
    };

    // Solve MdagM x = b.  `mat` is the high-precision operator, `matSloppy` the low-precision one (may be the same object).
    void invertCG(const Dirac &mat, const Dirac &matSloppy, ColorSpinorField &x, const ColorSpinorField &b, SolverParam &param);

    // ---- BiCGStab on M itself (behaviour of lib/inv_bicgstab_quda.cpp): the same precise / sloppy split and SolverParam;
    // restarts after a breakdown are counted in reliable_updates
    void invertBiCGStab(const Dirac &mat, const Dirac &matSloppy, ColorSpinorField &x, const ColorSpinorField &b, SolverParam &param);

    // ---- multi-shift CG on MdagM + sigma_j (behaviour of lib/inv_multi_cg_quda.cpp and the refinement of
    // invertMultiShiftQuda, lib/interface_quda.cpp:3580-3690)
    struct MultiShiftParam {
      int n_shift = 0;
      double offset[B200_MAX_SHIFTS] = {};     // non-decreasing
      double tol_offset[B200_MAX_SHIFTS] = {}; // per shift
      int maxiter = 10000;
      double delta = 0.1;
      // results
      int iter = 0;                              // multi-shift iterations
      int iter_offset[B200_MAX_SHIFTS] = {};     // iteration at which each shift retired
      int refine_iter[B200_MAX_SHIFTS] = {};     // iterations of each shift's refinement solve
      double iter_res_offset[B200_MAX_SHIFTS] = {};
      double true_res_offset[B200_MAX_SHIFTS] = {};
      int reliable_updates = 0;
      double secs = 0.0;
      double gflops = 0.0;
      int host_syncs = 0;
    };
    // throws unless 1 <= n_shift <= B200_MAX_SHIFTS, the offsets are finite and non-decreasing and every tol_offset > 0
    void checkMultiShiftParam(const MultiShiftParam &param);
    // Solve (MdagM + offset[j]) x_j = b for j < n_shift; x holds n_shift fields, which are overwritten
    void invertMultiShiftCG(const Dirac &mat, const Dirac &matSloppy, std::vector<ColorSpinorField> &x, const ColorSpinorField &b,
                            MultiShiftParam &param);

    // true if a halo wait gave up since the last call (clears the flag); the C entry points turn it into an error
    bool halo_timed_out(CommContext *comm, void *stream);

  } // namespace host
} // namespace b200
