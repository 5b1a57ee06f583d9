// Implementation of the host-side operator / blas / solver layer (design notes and reference citations: dirac.h).
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <cstdint>
#include <cstring>
#include <deque>
#include <map>
#include <memory>
#include <type_traits>
#include <cuda_runtime.h>

#include "dirac.h"

namespace b200
{
  namespace host
  {

    static void cuda_ok(cudaError_t e, const char *what)
    {
      if (e != cudaSuccess) throw Error(std::string(what) + ": " + cudaGetErrorString(e));
    }
    static void abi_ok(int rc)
    {
      if (rc != B200_SUCCESS) throw Error(b200_last_error());
    }
    static cudaStream_t cs(void *s) { return static_cast<cudaStream_t>(s); }

    // ------------------------------------------------------------------ fields
    static size_t parity_bytes_of(const int *X, int precision)
    {
      const size_t vcb = (size_t)X[0] * X[1] * X[2] * X[3] / 2;
      return vcb * 24 * precision + (precision == B200_HALF ? vcb * 4 : 0);
    }

    ColorSpinorField ColorSpinorField::wrap(void *v, const int *X, int precision, int n_parity)
    {
      ColorSpinorField f;
      f.v = v;
      for (int d = 0; d < 4; d++) f.X[d] = X[d];
      f.precision = precision;
      f.n_parity = n_parity;
      f.parity_bytes = parity_bytes_of(X, precision);
      return f;
    }

    ColorSpinorField ColorSpinorField::create(const int *X, int precision, int n_parity)
    {
      void *p = nullptr;
      const size_t bytes = parity_bytes_of(X, precision) * n_parity;
      cuda_ok(cudaMalloc(&p, bytes), "cudaMalloc(ColorSpinorField)");
      cuda_ok(cudaMemset(p, 0, bytes), "cudaMemset(ColorSpinorField)");
      ColorSpinorField f = wrap(p, X, precision, n_parity);
      f.owned = std::shared_ptr<void>(p, [](void *q) { cudaFree(q); });
      return f;
    }

    ColorSpinorField ColorSpinorField::parity_view(int p) const
    {
      if (n_parity != 2) throw Error("parity_view needs a full (two-parity) field");
      ColorSpinorField f = wrap(static_cast<char *>(v) + p * parity_bytes, X, precision, 1);
      f.owned = owned;
      return f;
    }

    b200_spinor ColorSpinorField::desc() const
    {
      b200_spinor s;
      s.v = v;
      s.norm = nullptr;
      s.parity_stride_bytes = n_parity == 2 ? parity_bytes : 0;
      s.volume_cb = VolumeCB();
      s.n_parity = n_parity;
      return s;
    }

    // Scratch fields: an operator application needs one or two temporaries; cudaMalloc per call would serialise the
    // device, so released temporaries are parked and reused -- per stream, because a parked buffer may still be read by
    // kernels queued on the stream that used it last.
    namespace
    {
      struct ScratchPool {
        std::multimap<void *, ColorSpinorField> parked; // keyed by stream
        ColorSpinorField get(void *stream, const int *X, int precision, int n_parity)
        {
          auto range = parked.equal_range(stream);
          for (auto it = range.first; it != range.second; ++it) {
            const ColorSpinorField &f = it->second;
            if (f.precision == precision && f.n_parity == n_parity && f.X[0] == X[0] && f.X[1] == X[1] && f.X[2] == X[2]
                && f.X[3] == X[3]) {
              ColorSpinorField r = f;
              parked.erase(it);
              return r;
            }
          }
          return ColorSpinorField::create(X, precision, n_parity);
        }
        void put(void *stream, const ColorSpinorField &f) { parked.emplace(stream, f); }
      };
      ScratchPool &pool()
      {
        static ScratchPool p;
        return p;
      }
      struct Scratch {
        void *stream;
        ColorSpinorField f;
        Scratch(void *stream_, const ColorSpinorField &like, int n_parity) :
          stream(stream_), f(pool().get(stream_, like.X, like.precision, n_parity))
        {
        }
        Scratch(void *stream_, const int *X, int precision, int n_parity) : stream(stream_), f(pool().get(stream_, X, precision, n_parity)) { }
        ~Scratch() { pool().put(stream, f); }
        operator ColorSpinorField &() { return f; }
      };

      // fork / join events of the two-stream halo schedule, one pair per halo context
      struct StreamEvents {
        cudaEvent_t fork = nullptr, join = nullptr;
      };
      StreamEvents &events_of(CommContext *c)
      {
        static std::map<CommContext *, StreamEvents> m;
        StreamEvents &e = m[c];
        if (!e.fork) {
          cuda_ok(cudaEventCreateWithFlags(&e.fork, cudaEventDisableTiming), "event");
          cuda_ok(cudaEventCreateWithFlags(&e.join, cudaEventDisableTiming), "event");
        }
        return e;
      }
    } // namespace

    // ------------------------------------------------------------------ Apply*
    static void halo_fill(b200_halo &h, const int *comm_override, CommContext *comm)
    {
      memset(&h, 0, sizeof(h));
      if (!comm) return;
      const unsigned seq = comm->seq();
      const int b = seq & 1;
      for (int d = 0; d < 4; d++) {
        h.comm_dim[d] = comm->comm_dim[d] && (!comm_override || comm_override[d]);
        for (int dir = 0; dir < 2; dir++) {
          h.ghost[d][dir] = h.comm_dim[d] ? comm->recv[b][d][dir] : nullptr;
          h.wait_flag[d][dir] = h.comm_dim[d] ? comm->recv_flag[b][d][dir] : nullptr;
        }
      }
      h.seq = seq;
      h.timeout_flag = comm->timeout_flag;
    }

    // describe the faces of `in` (single-parity field holding parity `in_parity`) and where they go; advances the exchange
    static void pack_args_for(b200_pack_args &a, const ColorSpinorField &in, int in_parity, bool dagger, const int *comm_override,
                              CommContext *comm)
    {
      const unsigned seq = ++comm->seq();
      const int b = seq & 1;
      memset(&a, 0, sizeof(a));
      a.abi_version = B200_ABI_VERSION;
      a.precision = in.precision;
      for (int d = 0; d < 4; d++) {
        a.X[d] = in.X[d];
        a.comm_dim[d] = comm->comm_dim[d] && (!comm_override || comm_override[d]);
        for (int f = 0; f < 2; f++) {
          a.dst[d][f] = comm->send_dst[b][d][f];
          a.signal[d][f] = comm->send_signal[b][d][f];
        }
      }
      a.parity = in_parity;
      a.dagger = dagger;
      a.in = in.desc();
      a.block_counter = comm->block_counter;
      a.seq = seq;
    }

    // two-stream schedule: ship the faces on the side stream
    static void exchange_start(const ColorSpinorField &in, int in_parity, bool dagger, const int *comm_override,
                               CommContext *comm, void *stream)
    {
      b200_pack_args a;
      pack_args_for(a, in, in_parity, dagger, comm_override, comm);
      if (comm->pack_stream && comm->pack_stream != stream) {
        // fork: the pack kernel runs on its own stream, concurrently with the interior tiles (joined in apply())
        StreamEvents &ev = events_of(comm);
        cuda_ok(cudaEventRecord(ev.fork, cs(stream)), "record");
        cuda_ok(cudaStreamWaitEvent(cs(comm->pack_stream), ev.fork, 0), "wait");
        a.stream = comm->pack_stream;
      } else {
        a.stream = stream;
      }
      abi_ok(b200_pack_ghost(&a));
    }

    // How a partitioned Dslash is issued (B200_HALO_SCHEDULE):
    //   split  two launches of dslash_fused_kernel: [pack | boundary] on the high-priority side stream, [interior] on the
    //          operator's stream, joined by an event (measured worst: the boundary CTAs spin from the start of the launch)
    //   fused  ONE launch [pack | interior | boundary] on the operator's stream (no side stream, no events)
    //   streams  the round-1 schedule: pack kernel + boundary-tile kernel on the side stream, interior tiles on the main one
    //   sites  as streams, but with 1-site-thick shells: pack kernel, then the boundary-site role on the side stream, the
    //          interior-site role on the main stream (18.75 % instead of 28 % of the sites take the branchy path at 8 GPUs)
    enum HaloSchedule { SCHED_AUTO = -1, SCHED_SPLIT = 0, SCHED_FUSED = 1, SCHED_STREAMS = 2, SCHED_SITES = 3 };
    // Default (B200_HALO_SCHEDULE unset): `streams` -- measured best at 2 and 8 GPUs for y/z/t splits -- unless x is
    // partitioned: tiles hold full x rows, so with an x split EVERY tile is a boundary tile and the tile-granular schedule has
    // no interior left to overlap with the halo (90.6 us at 2 GPUs); there the 1-site-thick shells of `sites` are used.
    static HaloSchedule halo_schedule(const int *comm_dim_eff)
    {
      static int v = -2;
      if (v == -2) {
        const char *e = getenv("B200_HALO_SCHEDULE");
        v = SCHED_AUTO;
        if (e && strcmp(e, "split") == 0) v = SCHED_SPLIT;
        if (e && strcmp(e, "fused") == 0) v = SCHED_FUSED;
        if (e && strcmp(e, "streams") == 0) v = SCHED_STREAMS;
        if (e && strcmp(e, "sites") == 0) v = SCHED_SITES;
      }
      if (v != SCHED_AUTO) return (HaloSchedule)v;
      return comm_dim_eff[0] ? SCHED_SITES : SCHED_STREAMS;
    }

    // `b`, `asymmetric`: twisted mass only; with_x: 1 / 0 force x on / off (the twisted-mass preconditioned operator's
    // xpay flag), -1 = the Wilson convention (x iff a != 0)
    static void apply(int op, ColorSpinorField &out, const ColorSpinorField &in, const GaugeField &U, const CloverField *A,
                      bool inverse_field, double a, const ColorSpinorField &x, int parity, bool dagger,
                      const int *comm_override, CommContext *comm, void *stream, double b = 0.0, bool asymmetric = false,
                      int with_x = -1)
    {
      if (in.precision != U.precision)
        throw Error("spinor precision " + std::to_string(in.precision) + " does not match the gauge field's " + std::to_string(U.precision));
      b200_dslash_args args;
      memset(&args, 0, sizeof(args));
      args.abi_version = B200_ABI_VERSION;
      args.op = op;
      args.kernel = B200_KERNEL_AUTO;
      args.precision = in.precision;
      for (int d = 0; d < 4; d++) args.X[d] = U.X[d];
      args.parity = parity == QUDA_INVALID_PARITY ? 0 : parity;
      args.dagger = dagger;
      args.a = a;
      args.out = out.desc();
      args.in = in.desc();
      if (with_x < 0 ? a != 0.0 : with_x != 0) args.x = x.desc();
      args.b = b;
      args.asymmetric = asymmetric ? 1 : 0;
      args.U = U.g;
      if (A) args.A = (inverse_field && A->has_inverse()) ? A->cinv : A->c;
      bool part = false;
      if (comm)
        for (int d = 0; d < 4; d++) part |= (comm->comm_dim[d] && (!comm_override || comm_override[d]));
      if (part && in.n_parity != 1) throw Error("a partitioned Dslash works on one parity at a time");
      const bool side_stream = part && comm->pack_stream && comm->pack_stream != stream;
      int eff[4] = {0, 0, 0, 0};
      if (part)
        for (int d = 0; d < 4; d++) eff[d] = comm->comm_dim[d] && (!comm_override || comm_override[d]);
      const HaloSchedule sched = part ? halo_schedule(eff) : SCHED_STREAMS;
      if (part && (sched == SCHED_FUSED || (sched == SCHED_SPLIT && !side_stream))) {
        // pack + interior + boundary: one launch on the operator's stream
        b200_pack_args pk;
        pack_args_for(pk, in, 1 - parity, dagger, comm_override, comm);
        pk.stream = stream;
        halo_fill(args.halo, comm_override, comm);
        args.stream = stream;
        abi_ok(b200_dslash_apply_fused(&args, &pk));
        return;
      }
      if (part && sched == SCHED_SPLIT) {
        // [pack | boundary] on the side stream (after `in` is complete), [interior] on the main stream, then join
        b200_pack_args pk;
        pack_args_for(pk, in, 1 - parity, dagger, comm_override, comm);
        halo_fill(args.halo, comm_override, comm);
        StreamEvents &ev = events_of(comm);
        cuda_ok(cudaEventRecord(ev.fork, cs(stream)), "record");
        cuda_ok(cudaStreamWaitEvent(cs(comm->pack_stream), ev.fork, 0), "wait");
        pk.stream = comm->pack_stream;
        args.stream = comm->pack_stream;
        args.kernel = B200_KERNEL_BOUNDARY_TILES;
        abi_ok(b200_dslash_apply_fused(&args, &pk));
        pk.stream = stream;
        args.stream = stream;
        args.kernel = B200_KERNEL_INTERIOR_TILES;
        abi_ok(b200_dslash_apply_fused(&args, &pk));
        cuda_ok(cudaEventRecord(ev.join, cs(comm->pack_stream)), "record");
        cuda_ok(cudaStreamWaitEvent(cs(stream), ev.join, 0), "wait");
        return;
      }
      if (part) exchange_start(in, 1 - parity, dagger, comm_override, comm, stream);
      halo_fill(args.halo, comm_override, part ? comm : nullptr);
      const bool two_streams = part && comm->pack_stream && comm->pack_stream != stream;
      if (two_streams) {
        // side stream (behind the pack kernel): boundary sites -- they depend only on the halo, not on the interior
        // launch; main stream: the interior.  Both halves write disjoint sites.
        const bool shells = sched == SCHED_SITES;
        args.kernel = shells ? B200_KERNEL_BOUNDARY_SITES : B200_KERNEL_BOUNDARY_TILES;
        args.stream = comm->pack_stream;
        abi_ok(b200_dslash_apply(&args));
        args.kernel = shells ? B200_KERNEL_INTERIOR_SITES : B200_KERNEL_INTERIOR_TILES;
        args.stream = stream;
        abi_ok(b200_dslash_apply(&args));
        // join: `out` is complete, and `in` may be overwritten, only after the side stream has drained
        StreamEvents &ev = events_of(comm);
        cuda_ok(cudaEventRecord(ev.join, cs(comm->pack_stream)), "record");
        cuda_ok(cudaStreamWaitEvent(cs(stream), ev.join, 0), "wait");
      } else {
        args.stream = stream;
        abi_ok(b200_dslash_apply(&args));
      }
    }

    void ApplyWilson(ColorSpinorField &out, const ColorSpinorField &in, const GaugeField &U, double a,
                     const ColorSpinorField &x, int parity, bool dagger, const int *comm_override, CommContext *comm,
                     void *stream)
    {
      apply(B200_OP_WILSON, out, in, U, nullptr, false, a, x, parity, dagger, comm_override, comm, stream);
    }

    void ApplyWilsonClover(ColorSpinorField &out, const ColorSpinorField &in, const GaugeField &U, const CloverField &A,
                           double a, const ColorSpinorField &x, int parity, bool dagger, const int *comm_override,
                           CommContext *comm, void *stream)
    {
      apply(B200_OP_CLOVER, out, in, U, &A, false, a, x, parity, dagger, comm_override, comm, stream);
    }

    void ApplyWilsonCloverPreconditioned(ColorSpinorField &out, const ColorSpinorField &in, const GaugeField &U,
                                         const CloverField &A, double a, const ColorSpinorField &x, int parity,
                                         bool dagger, const int *comm_override, CommContext *comm, void *stream)
    {
      apply(B200_OP_CLOVER_PC, out, in, U, &A, true, a, x, parity, dagger, comm_override, comm, stream);
    }

    void ApplyTwistedMass(ColorSpinorField &out, const ColorSpinorField &in, const GaugeField &U, double a, double b,
                          const ColorSpinorField &x, int parity, bool dagger, const int *comm_override, CommContext *comm,
                          void *stream)
    {
      apply(B200_OP_TWISTED_MASS, out, in, U, nullptr, false, a, x, parity, dagger, comm_override, comm, stream, b);
    }

    void ApplyTwistedMassPreconditioned(ColorSpinorField &out, const ColorSpinorField &in, const GaugeField &U, double a,
                                        double b, bool xpay, const ColorSpinorField &x, int parity, bool dagger,
                                        bool asymmetric, const int *comm_override, CommContext *comm, void *stream)
    {
      apply(B200_OP_TWISTED_MASS_PC, out, in, U, nullptr, false, a, x, parity, dagger, comm_override, comm, stream, b,
            asymmetric, xpay ? 1 : 0);
    }

    void ApplyTwistGamma(ColorSpinorField &out, const ColorSpinorField &in, double kappa, double mu, bool dagger, bool inverse,
                         void *stream)
    {
      b200_spinor o = out.desc(), i = in.desc();
      abi_ok(b200_twist_gamma5(&o, &i, in.precision, kappa, mu, dagger, inverse, stream));
    }

    void ApplyClover(ColorSpinorField &out, const ColorSpinorField &in, const CloverField &A, bool inverse, int parity,
                     void *stream)
    {
      b200_spinor o = out.desc(), i = in.desc();
      b200_clover c = (inverse && A.has_inverse()) ? A.cinv : A.c;
      abi_ok(b200_clover_apply(&o, &i, &c, in.precision, inverse, parity, stream));
    }

    bool halo_timed_out(CommContext *comm, void *stream)
    {
      if (!comm || !comm->timeout_flag) return false;
      int flag = 0;
      cuda_ok(cudaMemcpyAsync(&flag, comm->timeout_flag, sizeof(int), cudaMemcpyDeviceToHost, cs(stream)), "memcpy(timeout flag)");
      cuda_ok(cudaStreamSynchronize(cs(stream)), "sync");
      if (flag) cuda_ok(cudaMemsetAsync(comm->timeout_flag, 0, sizeof(int), cs(stream)), "memset(timeout flag)");
      return flag != 0;
    }

    // ------------------------------------------------------------------ blas + reductions
    namespace blas
    {
      static long long g_flops = 0;
      long long flops() { return g_flops; }

      constexpr int kBlocks = 132 * 4, kThreads = 256, kMaxVals = 2;

      // device-resident scalars of a solve (read by the update kernels, written by the reduction finalisers)
      enum Scalar { S_R2 = 0, S_R2_OLD = 1, S_PAP = 2, S_ALPHA = 3, S_BETA = 4, S_RAW0 = 5, S_RAW1 = 6, S_COUNT = 8 };
      enum Finish { FIN_RAW = 0, FIN_PAP = 1, FIN_R2 = 2 };

      // NVLink mailboxes of the all-reduce (b200_comm::reduce_peer): slot [parity of seq][source rank] in every rank's box
      struct ReduceSlot {
        double v[4];
        unsigned seq;
        unsigned pad[7];
      };
      static_assert(sizeof(ReduceSlot) == B200_REDUCE_SLOT_BYTES, "mailbox slot layout");
      struct ReducePeers {
        ReduceSlot *box[B200_MAX_RANKS];
        int rank, n_ranks;
        unsigned seq;
        int *timeout_flag;
      };

      // Derive CG's scalars from the global sums in S[S_RAW0..]: on the device in the last block of a reduction, or on the
      // host after the host all-reduce (no NVLink mailboxes).
      //   FIN_PAP  v = <p, Ap>    pAp <- v, alpha = r2 / v
      //   FIN_R2   v = |r|^2      r2_old <- r2, r2 <- v, beta = v / r2_old
      __host__ __device__ inline void cg_scalars(double *S, int fin)
      {
        const double v0 = S[S_RAW0];
        if (fin == FIN_PAP) {
          S[S_PAP] = v0;
          S[S_ALPHA] = S[S_R2] / v0;
        } else if (fin == FIN_R2) {
          const double old = S[S_R2];
          S[S_R2_OLD] = old;
          S[S_R2] = v0;
          S[S_BETA] = v0 / old;
        }
      }
      // A solver's scalar block: sums per reduction (kVals), block size (kCount), where the raw sums go (kRaw), and the
      // function that derives the scalars from them.  Finaliser 0 (FIN_RAW, BF_RAW) only stores the sums.
      struct CgTraits {
        static constexpr int kVals = kMaxVals, kCount = S_COUNT, kRaw = S_RAW0;
        __host__ __device__ static void derive(double *S, int fin) { cg_scalars(S, fin); }
      };

      // per-stream reduction workspace of one solver's scalar block
      struct Workspace {
        double *partials = nullptr; // [kBlocks][kVals]
        unsigned *ticket = nullptr;
        double *scalars = nullptr;  // [kCount] on the device
        double *host = nullptr;     // pinned + mapped: [ring][kCount], written by the finalisers
        double *host_dev = nullptr; // device alias of `host`
        cudaEvent_t ev[8] = {};
        unsigned long long ring = 0;
      };
      template <typename Tr> static Workspace &workspace(void *stream)
      {
        static std::map<void *, Workspace> m;
        Workspace &w = m[stream];
        if (!w.partials) {
          cuda_ok(cudaMalloc(&w.partials, sizeof(double) * kBlocks * Tr::kVals), "cudaMalloc(reduce)");
          cuda_ok(cudaMalloc(&w.ticket, sizeof(unsigned)), "cudaMalloc(reduce)");
          cuda_ok(cudaMemset(w.ticket, 0, sizeof(unsigned)), "memset");
          cuda_ok(cudaMalloc(&w.scalars, sizeof(double) * Tr::kCount), "cudaMalloc(reduce)");
          cuda_ok(cudaMemset(w.scalars, 0, sizeof(double) * Tr::kCount), "memset");
          cuda_ok(cudaHostAlloc(&w.host, sizeof(double) * 8 * Tr::kCount, cudaHostAllocMapped), "cudaHostAlloc(reduce)");
          cuda_ok(cudaHostGetDevicePointer(&w.host_dev, w.host, 0), "cudaHostGetDevicePointer");
          for (auto &e : w.ev) cuda_ok(cudaEventCreateWithFlags(&e, cudaEventDisableTiming), "event");
        }
        return w;
      }

      // Second stage of every reduction, run by the block that arrives last: sum the per-block partial sums in block
      // order (fixed -> bit-reproducible), all-reduce over the ranks through the NVLink mailboxes in rank order, store the
      // global sums in the raw slots, derive the solver's scalars and publish the scalar block to the host mirror.
      struct ReduceArgs {
        double *partials; // [kBlocks][Tr::kVals]
        unsigned *ticket;
        double *S;        // the solver's scalar block
        double *host_out; // its mirror slot, or null
        int fin;          // the finaliser: what Tr::derive computes from the sums
        ReducePeers peers;
      };
      template <int NV, typename Tr> __device__ void finish_reduction(const double *acc_block, const ReduceArgs &ra)
      {
        constexpr int MV = Tr::kVals;
        __shared__ double sh[kThreads][MV];
        __shared__ bool is_last;
        __shared__ double part[B200_MAX_RANKS][MV];
        // copies of the arguments: reading them in place, peers above all, gives the finalisers another schedule
        double *partials = ra.partials, *S = ra.S, *host_out = ra.host_out;
        unsigned *ticket = ra.ticket;
        const int fin = ra.fin;
        const ReducePeers peers = ra.peers;
        const int t = threadIdx.x;
        if (t == 0) {
          for (int i = 0; i < NV; i++) partials[blockIdx.x * MV + i] = acc_block[i];
          __threadfence();
          is_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
        }
        __syncthreads();
        if (!is_last) return;
        __threadfence();
        double a[MV] = {};
        for (int b = t; b < (int)gridDim.x; b += kThreads)
          for (int i = 0; i < NV; i++) a[i] += __ldcg(partials + b * MV + i);
        for (int i = 0; i < NV; i++) sh[t][i] = a[i];
        __syncthreads();
        for (int s = kThreads / 2; s > 0; s >>= 1) {
          if (t < s)
            for (int i = 0; i < NV; i++) sh[t][i] += sh[t + s][i];
          __syncthreads();
        }
        if (peers.n_ranks > 1) {
          const int b = peers.seq & 1;
          if (t < peers.n_ranks) {
            ReduceSlot *dst = peers.box[t] + b * B200_MAX_RANKS + peers.rank;
            for (int i = 0; i < NV; i++) dst->v[i] = sh[0][i];
            __threadfence_system();
            asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(&dst->seq), "r"(peers.seq) : "memory");
            const ReduceSlot *src = peers.box[peers.rank] + b * B200_MAX_RANKS + t;
            const long long t0 = clock64();
            for (;;) {
              unsigned got;
              asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(got) : "l"(&src->seq) : "memory");
              if ((int)(got - peers.seq) >= 0) break;
              if (clock64() - t0 > 20000000000LL) { // ~10 s: a lost peer must never hang the GPU
                if (peers.timeout_flag) *peers.timeout_flag = 1;
                break;
              }
              __nanosleep(40);
            }
            for (int i = 0; i < NV; i++) part[t][i] = *reinterpret_cast<const volatile double *>(&src->v[i]);
          }
          __syncthreads();
          if (t == 0)
            for (int i = 0; i < NV; i++) {
              double s = 0;
              for (int r = 0; r < peers.n_ranks; r++) s += part[r][i];
              sh[0][i] = s;
            }
        }
        if (t == 0) {
          for (int i = 0; i < NV; i++) S[Tr::kRaw + i] = sh[0][i];
          Tr::derive(S, fin);
          if (host_out) {
            for (int i = 0; i < Tr::kCount; i++) host_out[i] = S[i];
            __threadfence_system();
          }
          *ticket = 0;
        }
      }

      __device__ __forceinline__ double warp_sum(double v)
      {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
        return v;
      }
      // per-block sum of per-thread values, in a fixed order (warp tree, then warps in index order)
      __device__ __forceinline__ double block_sum(double v, double *warp_buf)
      {
        v = warp_sum(v);
        const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
        if (l == 0) warp_buf[w] = v;
        __syncthreads();
        double s = 0;
        if (threadIdx.x == 0)
          for (int i = 0; i < kThreads / 32; i++) s += warp_buf[i];
        __syncthreads();
        return s;
      }
      // the tail of every reduction kernel: the block sum of each per-thread value, then the second stage
      template <typename Tr, int NV> __device__ __forceinline__ void reduce_block(const double (&acc)[NV], const ReduceArgs &ra)
      {
        __shared__ double wb[kThreads / 32];
        double s[NV];
#pragma unroll
        for (int i = 0; i < NV; i++) s[i] = block_sum(acc[i], wb);
        finish_reduction<NV, Tr>(s, ra);
      }

      // y = a x + b y with an optional reduction over the result (R_NORM_Y) or <x, y> (R_DOT_XY)
      enum { R_NONE = 0, R_NORM_Y = 1, R_DOT_XY = 2 };
      template <typename Tx, typename Ty, int R>
      __global__ void __launch_bounds__(kThreads) axpby_kernel(double a, const Tx *__restrict__ x, double b, Ty *__restrict__ y,
                                                               size_t n, bool write, ReduceArgs ra)
      {
        double acc = 0;
        for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
          const double xv = x[i], yv = y[i];
          const double r = a * xv + b * yv;
          if (write) y[i] = (Ty)r;
          if (R == R_NORM_Y) acc += (write ? (double)(Ty)r * (double)(Ty)r : yv * yv);
          if (R == R_DOT_XY) acc += xv * yv;
        }
        if (R != R_NONE) reduce_block<CgTraits>({acc}, ra);
      }

      // ---- the three kernels of a CG iteration; alpha and beta come from the device scalars
      // r -= alpha Ap ; |r|^2   (finaliser: r2_old <- r2, r2 <- |r|^2, beta <- r2 / r2_old)
      template <typename T>
      __global__ void __launch_bounds__(kThreads) cg_update_r_kernel(T *__restrict__ r, const T *__restrict__ Ap, size_t n, ReduceArgs ra)
      {
        const double alpha = ra.S[S_ALPHA];
        double acc = 0;
        for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
          const T v = (T)((double)r[i] - alpha * (double)Ap[i]);
          r[i] = v;
          acc += (double)v * (double)v;
        }
        reduce_block<CgTraits>({acc}, ra);
      }
      // x += alpha p ; p = r + beta p   (the reference's axpyZpbx, lib/inv_cg_quda.cpp:389)
      template <typename T>
      __global__ void __launch_bounds__(kThreads) cg_update_xp_kernel(T *__restrict__ x, T *__restrict__ p, const T *__restrict__ r,
                                                                      size_t n, const double *__restrict__ S)
      {
        const double alpha = S[S_ALPHA], beta = S[S_BETA];
        for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
          const double pv = p[i];
          x[i] = (T)((double)x[i] + alpha * pv);
          p[i] = (T)((double)r[i] + beta * pv);
        }
      }
      // after a reliable update: p += r_new - r_old ; r_old <- r_new   (keeps p = r + beta p_old with the true residual)
      template <typename T>
      __global__ void __launch_bounds__(kThreads) cg_replace_r_kernel(T *__restrict__ p, T *__restrict__ r, const T *__restrict__ r_new, size_t n)
      {
        for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
          const T rn = r_new[i];
          p[i] = (T)((double)p[i] + ((double)rn - (double)r[i]));
          r[i] = rn;
        }
      }
      __global__ void set_scalar_kernel(double *S, int idx, double v) { S[idx] = v; }

      // ---- BiCGStab: its own device scalar block (complex scalars are (re, im) pairs) and finalisers
      enum BicgScalar {
        B_RHO = 0, B_ALPHA = 2, B_OMEGA = 4, B_BETA = 6, B_R2 = 8, B_STOP = 9,
        B_DONE = 10,  // 1 once |r|^2 <= stop: every BiCGStab kernel after that returns at once, until the host clears it
        B_BREAK = 11, // breakdown word (BRK_* bits): a zero divisor met while the residual was not 0
        B_RAW = 12,   // the global sums of the last reduction, up to 4
        B_COUNT = 16
      };
      enum BicgFinish { BF_RAW = FIN_RAW, BF_RHO = 1, BF_ALPHA = 2, BF_OMEGA = 3, BF_BETA = 4 };
      enum { BRK_ALPHA = 1, BRK_OMEGA = 2, BRK_BETA = 4 };

      // rounded products: no FMA contraction, so that (a + ib) / (a + ib) is exactly 1 on the device and on the host
      __host__ __device__ inline double mul_rn(double a, double b)
      {
#ifdef __CUDA_ARCH__
        return __dmul_rn(a, b);
#else
        return a * b;
#endif
      }
      // q = n / d, or 0 if d == 0 (returns false then)
      __host__ __device__ inline bool cdiv(double *q, double nr, double ni, double dr, double di)
      {
        const double den = mul_rn(dr, dr) + mul_rn(di, di);
        if (den == 0.0) {
          q[0] = q[1] = 0.0;
          return false;
        }
        q[0] = (mul_rn(nr, dr) + mul_rn(ni, di)) / den;
        q[1] = (mul_rn(ni, dr) - mul_rn(nr, di)) / den;
        return true;
      }
      __host__ __device__ inline void cmul(double *q, double ar, double ai, double br, double bi)
      {
        const double re = mul_rn(ar, br) - mul_rn(ai, bi), im = mul_rn(ar, bi) + mul_rn(ai, br);
        q[0] = re;
        q[1] = im;
      }
      // a zero divisor is a breakdown unless the residual the step leaves behind is 0 (that is convergence)
      __host__ __device__ inline void breakdown(double *S, int bit, double r2_left)
      {
        if (r2_left != 0.0) S[B_BREAK] = (double)((int)S[B_BREAK] | bit);
      }
      // Derive BiCGStab's scalars from the global sums in S[B_RAW..]: on the device in the last block of a reduction, or on
      // the host after the host all-reduce (no NVLink mailboxes).
      //   BF_RHO    v = <r0, r>                 rho <- v
      //   BF_ALPHA  v = <r0, v>                 alpha = rho / v            (0 if v == 0)
      //   BF_OMEGA  v = <t, s>, |t|^2, |s|^2    omega = <t, s> / |t|^2     (0 if |t|^2 == 0; s is then left as r)
      //   BF_BETA   v = <r0, r>, |r|^2          beta = (v / rho)(alpha / omega) (0 if omega or rho is 0), rho <- v, r2 <- |r|^2
      __host__ __device__ inline void bicg_scalars(double *S, int fin)
      {
        const double *v = S + B_RAW;
        if (fin == BF_RHO) {
          S[B_RHO] = v[0];
          S[B_RHO + 1] = v[1];
        } else if (fin == BF_ALPHA) {
          if (!cdiv(S + B_ALPHA, S[B_RHO], S[B_RHO + 1], v[0], v[1])) breakdown(S, BRK_ALPHA, S[B_R2]);
        } else if (fin == BF_OMEGA) {
          if (v[2] == 0.0) {
            S[B_OMEGA] = S[B_OMEGA + 1] = 0.0;
            breakdown(S, BRK_OMEGA, v[3]);
          } else {
            S[B_OMEGA] = v[0] / v[2];
            S[B_OMEGA + 1] = v[1] / v[2];
          }
        } else if (fin == BF_BETA) {
          double q[2], a[2];
          const bool ok = cdiv(q, v[0], v[1], S[B_RHO], S[B_RHO + 1]) && cdiv(a, S[B_ALPHA], S[B_ALPHA + 1], S[B_OMEGA], S[B_OMEGA + 1]);
          if (ok) {
            cmul(S + B_BETA, q[0], q[1], a[0], a[1]);
          } else {
            S[B_BETA] = S[B_BETA + 1] = 0.0;
            breakdown(S, BRK_BETA, v[2]);
          }
          S[B_RHO] = v[0];
          S[B_RHO + 1] = v[1];
          S[B_R2] = v[2];
          if (v[2] <= S[B_STOP]) S[B_DONE] = 1.0;
        }
      }
      struct BicgTraits {
        static constexpr int kVals = 4, kCount = B_COUNT, kRaw = B_RAW;
        __host__ __device__ static void derive(double *S, int fin) { bicg_scalars(S, fin); }
      };

      template <typename T> using Cplx = std::conditional_t<std::is_same<T, double>::value, double2, float2>;

      // The five streaming kernels of a BiCGStab iteration walk the field as complex numbers: in both native orders (fp64
      // planes of 2 reals, fp32 planes of 4) the real index 2c + re/im keeps each pair adjacent, so element pair i is one
      // complex component.  n is the number of complex elements.  Every kernel returns at once when S[B_DONE] is set.

      // K1 (and the rho (re)computation): <a, b> = sum conj(a) b
      template <typename T>
      __global__ void __launch_bounds__(kThreads) bicg_cdot_kernel(const T *__restrict__ a_, const T *__restrict__ b_, size_t n, ReduceArgs ra)
      {
        using C2 = Cplx<T>;
        if (ra.S[B_DONE] != 0.0) return;
        const C2 *a = reinterpret_cast<const C2 *>(a_), *b = reinterpret_cast<const C2 *>(b_);
        double acc[2] = {0, 0};
        for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
          const C2 x = a[i], y = b[i];
          acc[0] += (double)x.x * y.x + (double)x.y * y.y;
          acc[1] += (double)x.x * y.y - (double)x.y * y.x;
        }
        reduce_block<BicgTraits>(acc, ra);
      }
      // K2: s = r - alpha v, in place in r
      template <typename T>
      __global__ void __launch_bounds__(kThreads) bicg_update_s_kernel(T *__restrict__ r_, const T *__restrict__ v_, size_t n, const double *__restrict__ S)
      {
        using C2 = Cplx<T>;
        if (S[B_DONE] != 0.0) return;
        const double ar = S[B_ALPHA], ai = S[B_ALPHA + 1];
        C2 *r = reinterpret_cast<C2 *>(r_);
        const C2 *v = reinterpret_cast<const C2 *>(v_);
        for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
          const C2 x = v[i], y = r[i];
          C2 o;
          o.x = (T)((double)y.x - (ar * x.x - ai * x.y));
          o.y = (T)((double)y.y - (ar * x.y + ai * x.x));
          r[i] = o;
        }
      }
      // K3: <t, s>, |t|^2, |s|^2
      template <typename T>
      __global__ void __launch_bounds__(kThreads) bicg_ts_kernel(const T *__restrict__ t_, const T *__restrict__ s_, size_t n, ReduceArgs ra)
      {
        using C2 = Cplx<T>;
        if (ra.S[B_DONE] != 0.0) return;
        const C2 *t = reinterpret_cast<const C2 *>(t_), *s = reinterpret_cast<const C2 *>(s_);
        double acc[4] = {0, 0, 0, 0};
        for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
          const C2 x = t[i], y = s[i];
          acc[0] += (double)x.x * y.x + (double)x.y * y.y;
          acc[1] += (double)x.x * y.y - (double)x.y * y.x;
          acc[2] += (double)x.x * x.x + (double)x.y * x.y;
          acc[3] += (double)y.x * y.x + (double)y.y * y.y;
        }
        reduce_block<BicgTraits>(acc, ra);
      }
      // K4: x += alpha p + omega s ; r = s - omega t (r holds s) ; <r0, r>, |r|^2 of the stored r
      template <typename T>
      __global__ void __launch_bounds__(kThreads) bicg_update_xr_kernel(T *__restrict__ x_, T *__restrict__ r_, const T *__restrict__ p_,
                                                                        const T *__restrict__ t_, const T *__restrict__ r0_, size_t n, ReduceArgs ra)
      {
        using C2 = Cplx<T>;
        const double *S = ra.S;
        if (S[B_DONE] != 0.0) return;
        const double ar = S[B_ALPHA], ai = S[B_ALPHA + 1], wr = S[B_OMEGA], wi = S[B_OMEGA + 1];
        C2 *x = reinterpret_cast<C2 *>(x_), *r = reinterpret_cast<C2 *>(r_);
        const C2 *p = reinterpret_cast<const C2 *>(p_), *t = reinterpret_cast<const C2 *>(t_), *r0 = reinterpret_cast<const C2 *>(r0_);
        double acc[3] = {0, 0, 0};
        for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
          const C2 pv = p[i], sv = r[i], tv = t[i], xv = x[i], hv = r0[i];
          C2 xo, ro;
          xo.x = (T)((double)xv.x + (ar * pv.x - ai * pv.y) + (wr * sv.x - wi * sv.y));
          xo.y = (T)((double)xv.y + (ar * pv.y + ai * pv.x) + (wr * sv.y + wi * sv.x));
          ro.x = (T)((double)sv.x - (wr * tv.x - wi * tv.y));
          ro.y = (T)((double)sv.y - (wr * tv.y + wi * tv.x));
          x[i] = xo;
          r[i] = ro;
          acc[0] += (double)hv.x * ro.x + (double)hv.y * ro.y;
          acc[1] += (double)hv.x * ro.y - (double)hv.y * ro.x;
          acc[2] += (double)ro.x * ro.x + (double)ro.y * ro.y;
        }
        reduce_block<BicgTraits>(acc, ra);
      }
      // K5: p = r + beta (p - omega v)
      template <typename T>
      __global__ void __launch_bounds__(kThreads) bicg_update_p_kernel(T *__restrict__ p_, const T *__restrict__ r_, const T *__restrict__ v_,
                                                                       size_t n, const double *__restrict__ S)
      {
        using C2 = Cplx<T>;
        if (S[B_DONE] != 0.0) return;
        const double br = S[B_BETA], bi = S[B_BETA + 1], wr = S[B_OMEGA], wi = S[B_OMEGA + 1];
        C2 *p = reinterpret_cast<C2 *>(p_);
        const C2 *r = reinterpret_cast<const C2 *>(r_), *v = reinterpret_cast<const C2 *>(v_);
        for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
          const C2 pv = p[i], rv = r[i], vv = v[i];
          const double dr = pv.x - (wr * vv.x - wi * vv.y), di = pv.y - (wr * vv.y + wi * vv.x);
          C2 o;
          o.x = (T)((double)rv.x + (br * dr - bi * di));
          o.y = (T)((double)rv.y + (br * di + bi * dr));
          p[i] = o;
        }
      }
      template <int N> struct Scalars {
        double s[N];
      };
      // the whole scalar block of a solver (one thread per scalar)
      template <int N> __global__ void set_scalars_kernel(double *S, Scalars<N> v)
      {
        if (threadIdx.x < N) S[threadIdx.x] = v.s[threadIdx.x];
      }

      // ---- multi-shift CG: one scalar block for all shifts.  Per-shift arrays of B200_MAX_SHIFTS entries; shift 0 is the
      // unshifted recursion (zeta_0 = 1, alpha_0 / beta_0 are CG's alpha / beta).  The active shifts are always the prefix
      // j < M_NACT: a shift retires only after every shift above it has.
      constexpr int kShifts = B200_MAX_SHIFTS;
      enum MsScalar {
        M_R2 = 0, M_R2_OLD = 1, M_PAP = 2,
        M_NACT = 3,    // active shifts
        M_NUPD = 4,    // shifts the x / p update of this iteration touches (M_NACT before this iteration's retirements)
        M_DONE = 5,    // 1 once every shift has retired: every multi-shift kernel after that returns at once
        M_ITER = 6,    // iterations completed (|r|^2 finalisers run)
        M_RAW = 7,     // the global sum of the last reduction
        M_DSIG = 16,                   // sigma_j - sigma_0
        M_ZETA = M_DSIG + kShifts,     // zeta_j
        M_ZOLD = M_ZETA + kShifts,     // zeta_j of the previous iteration
        M_ALPHA = M_ZOLD + kShifts,    // alpha_j
        M_BETA = M_ALPHA + kShifts,    // beta_j
        M_STOP = M_BETA + kShifts,     // stopping value of |r_j|^2
        M_RES = M_STOP + kShifts,      // |r_j|^2 = zeta_j^2 |r|^2, frozen when shift j retires
        M_RETIRED = M_RES + kShifts,   // iteration at which shift j retired (-1: still active)
        M_COUNT = M_RETIRED + kShifts
      };
      // Derive the multi-shift scalars from the global sum in S[M_RAW] (the CG-M recursion, lib/inv_multi_cg_quda.cpp):
      //   FIN_PAP  v = <p_0, (A + sigma_0) p_0>   alpha_0 = r2 / v; for the active shifts zeta_j, zeta_old_j, alpha_j
      //                                          (updateAlphaZeta, :170-186); M_NUPD <- M_NACT
      //   FIN_R2   v = |r|^2                     r2_old <- r2, r2 <- v, beta_0 = v / r2_old,
      //                                          beta_j = beta_0 zeta_j alpha_j / (zeta_old_j alpha_0) (:100, :380); then retire
      //                                          shifts from the top while zeta_j^2 r2 <= stop_j (:394-409), done when none is left
      // Zero divisors give zero, never NaN; a shift with zeta_j = 0 has converged.  Products are rounded one by one
      // (mul_rn), so the device and the host derive bit-identical scalars.
      __host__ __device__ inline void ms_scalars(double *S, int fin)
      {
        double *dsig = S + M_DSIG, *zeta = S + M_ZETA, *zold = S + M_ZOLD, *alpha = S + M_ALPHA, *beta = S + M_BETA;
        const double v = S[M_RAW];
        int n = (int)S[M_NACT];
        if (fin == FIN_PAP) {
          const double a_old = alpha[0], b_old = beta[0];
          const double a0 = v != 0.0 ? S[M_R2] / v : 0.0;
          S[M_PAP] = v;
          alpha[0] = a0;
          for (int j = 1; j < n; j++) {
            const double c0 = mul_rn(mul_rn(zeta[j], zold[j]), a_old);
            const double c1 = mul_rn(mul_rn(a0, b_old), zold[j] - zeta[j]);
            const double c2 = mul_rn(mul_rn(zold[j], a_old), 1.0 + mul_rn(dsig[j], a0));
            const double den = c1 + c2;
            zold[j] = zeta[j];
            zeta[j] = den != 0.0 ? c0 / den : 0.0;
            alpha[j] = zeta[j] != 0.0 ? mul_rn(a0, zeta[j]) / zold[j] : 0.0; // zeta_j != 0 needs c0 != 0, so zold_j != 0
          }
          S[M_NUPD] = n;
        } else if (fin == FIN_R2) {
          const double old = S[M_R2];
          S[M_R2_OLD] = old;
          S[M_R2] = v;
          const double b0 = old != 0.0 ? v / old : 0.0;
          beta[0] = b0;
          for (int j = 1; j < n; j++) {
            const double den = mul_rn(zold[j], alpha[0]);
            beta[j] = den != 0.0 ? mul_rn(mul_rn(b0, zeta[j]), alpha[j]) / den : 0.0;
          }
          S[M_ITER] += 1.0;
          for (int j = 0; j < n; j++) S[M_RES + j] = mul_rn(mul_rn(zeta[j], zeta[j]), v);
          while (n > 0 && S[M_RES + n - 1] <= S[M_STOP + n - 1]) {
            n--;
            S[M_RETIRED + n] = S[M_ITER];
          }
          S[M_NACT] = n;
          if (n == 0) S[M_DONE] = 1.0;
        }
      }
      struct MsTraits {
        static constexpr int kVals = 1, kCount = M_COUNT, kRaw = M_RAW;
        __host__ __device__ static void derive(double *S, int fin) { ms_scalars(S, fin); }
      };

      // The multi-shift kernels move 16 bytes per access: 2 doubles or 4 floats.  Both native orders keep the field a
      // flat array of reals and the kernels act element-wise, so element i of every field is the same component.
      template <typename T> struct alignas(16) Vec {
        static constexpr int W = 16 / sizeof(T);
        T e[W];
      };
      // the x and p fields of every shift, by value
      template <typename T> struct MsFields {
        T *x[kShifts];
        T *p[kShifts];
      };
      // Ap += sigma_0 p ; <p, Ap>   (finaliser FIN_PAP).  Once M_DONE is set it returns at once, and clears M_NUPD so
      // that the x / p update queued behind it does nothing either.
      template <typename T>
      __global__ void __launch_bounds__(kThreads) ms_dot_kernel(const Vec<T> *__restrict__ p, Vec<T> *__restrict__ Ap, double sigma,
                                                                size_t n, ReduceArgs ra)
      {
        if (ra.S[M_DONE] != 0.0) {
          if (blockIdx.x == 0 && threadIdx.x == 0) ra.S[M_NUPD] = 0.0;
          return;
        }
        double acc = 0;
        for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
          const Vec<T> pv = p[i];
          Vec<T> av = Ap[i];
#pragma unroll
          for (int e = 0; e < Vec<T>::W; e++) {
            av.e[e] = (T)((double)av.e[e] + sigma * (double)pv.e[e]);
            acc += (double)pv.e[e] * (double)av.e[e];
          }
          if (sigma != 0.0) Ap[i] = av;
        }
        reduce_block<MsTraits>({acc}, ra);
      }
      // r -= alpha_0 Ap ; |r|^2   (finaliser FIN_R2: beta_j, retirement, done flag)
      template <typename T>
      __global__ void __launch_bounds__(kThreads) ms_update_r_kernel(Vec<T> *__restrict__ r, const Vec<T> *__restrict__ Ap, size_t n,
                                                                     ReduceArgs ra)
      {
        if (ra.S[M_DONE] != 0.0) return;
        const double alpha = ra.S[M_ALPHA];
        double acc = 0;
        for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
          const Vec<T> av = Ap[i];
          Vec<T> rv = r[i];
#pragma unroll
          for (int e = 0; e < Vec<T>::W; e++) {
            rv.e[e] = (T)((double)rv.e[e] - alpha * (double)av.e[e]);
            acc += (double)rv.e[e] * (double)rv.e[e];
          }
          r[i] = rv;
        }
        reduce_block<MsTraits>({acc}, ra);
      }
      // The hot path: for every shift j < M_NUPD, x_j += alpha_j p_j ; p_j = zeta_j r + beta_j p_j (shift 0: zeta = 1, the
      // reference's axpyZpbx; the others its axpyBzpcx).  r is read once per element; a retired shift costs no bytes:
      // (1 + 4 M_NUPD) fields of traffic.
      template <typename T>
      __global__ void __launch_bounds__(kThreads) ms_update_xp_kernel(MsFields<T> f, const Vec<T> *__restrict__ r, size_t n,
                                                                      const double *__restrict__ S)
      {
        __shared__ double c[3][kShifts]; // alpha_j, zeta_j, beta_j
        const int ns = (int)S[M_NUPD];
        if (ns == 0) return;
        const int t = threadIdx.x;
        if (t < ns) {
          c[0][t] = S[M_ALPHA + t];
          c[1][t] = S[M_ZETA + t];
          c[2][t] = S[M_BETA + t];
        }
        __syncthreads();
        for (size_t i = (size_t)blockIdx.x * blockDim.x + t; i < n; i += (size_t)gridDim.x * blockDim.x) {
          const Vec<T> rv = r[i];
          for (int j = 0; j < ns; j++) {
            Vec<T> *x = reinterpret_cast<Vec<T> *>(f.x[j]), *p = reinterpret_cast<Vec<T> *>(f.p[j]);
            const double a = c[0][j], z = c[1][j], b = c[2][j];
            Vec<T> xv = x[i], pv = p[i];
#pragma unroll
            for (int e = 0; e < Vec<T>::W; e++) {
              const double pe = pv.e[e];
              xv.e[e] = (T)((double)xv.e[e] + a * pe);
              pv.e[e] = (T)(z * (double)rv.e[e] + b * pe);
            }
            x[i] = xv;
            p[i] = pv;
          }
        }
      }
      // After a reliable update: d = r_new - r ; p_0 += d, p_j += zeta_j d for the active shifts ; r = r_new.  That keeps
      // p_j = zeta_j r_new + beta_j p_j,old exactly (CG's late-update repair, per shift).  It also stores the true |r|^2,
      // clears M_DONE and reopens shift 0 if every shift had retired; the blocks that read M_NACT before or after
      // block 0 rewrites it get the same count.
      template <typename T>
      __global__ void __launch_bounds__(kThreads) ms_replace_r_kernel(MsFields<T> f, Vec<T> *__restrict__ r, const Vec<T> *__restrict__ r_new,
                                                                      size_t n, double *S, double r2)
      {
        __shared__ double z[kShifts];
        const int ns = max((int)S[M_NACT], 1);
        const int t = threadIdx.x;
        if (t < ns) z[t] = t == 0 ? 1.0 : S[M_ZETA + t];
        __syncthreads();
        if (blockIdx.x == 0 && t == 0) {
          S[M_NACT] = ns;
          S[M_DONE] = 0.0;
          S[M_R2] = r2;
        }
        for (size_t i = (size_t)blockIdx.x * blockDim.x + t; i < n; i += (size_t)gridDim.x * blockDim.x) {
          const Vec<T> rn = r_new[i], ro = r[i];
          for (int j = 0; j < ns; j++) {
            Vec<T> *p = reinterpret_cast<Vec<T> *>(f.p[j]);
            Vec<T> pv = p[i];
#pragma unroll
            for (int e = 0; e < Vec<T>::W; e++) pv.e[e] = (T)((double)pv.e[e] + z[j] * ((double)rn.e[e] - (double)ro.e[e]));
            p[i] = pv;
          }
          r[i] = rn;
        }
      }

      static void check_pair(const ColorSpinorField &x, const ColorSpinorField &y)
      {
        if (x.Length() != y.Length()) throw Error("blas: operands differ in length");
        if (x.precision == B200_HALF || y.precision == B200_HALF) throw Error("blas: half-precision (block-float) fields are not supported");
      }
      template <typename... F> static void check_same(const ColorSpinorField &x, const F &...ys)
      {
        for (const ColorSpinorField *y : {&ys...}) {
          check_pair(x, *y);
          if (x.precision != y->precision) throw Error("blas: operands differ in precision (convert with blas::copy)");
        }
      }

      // Calls f(T()) with T = double for fp64 fields and float for fp32 ones (f launches the kernel instantiated for T),
      // then checks the launch and counts its flops.
      template <typename F> static void launch(int precision, long long flops, F &&f)
      {
        if (precision == 8) f(double());
        else f(float());
        cuda_ok(cudaGetLastError(), "blas launch");
        g_flops += flops;
      }

      static ReducePeers peers_of(CommContext *comm)
      {
        ReducePeers p;
        memset(&p, 0, sizeof(p));
        p.n_ranks = 1;
        if (comm && comm->mailboxes()) {
          if (comm->n_ranks > B200_MAX_RANKS) throw Error("NVLink all-reduce: more ranks than mailbox slots");
          for (int r = 0; r < B200_MAX_RANKS; r++) p.box[r] = reinterpret_cast<ReduceSlot *>(comm->reduce_peer[r]);
          p.rank = comm->rank;
          p.n_ranks = comm->n_ranks;
          p.seq = ++comm->reduce_seq();
          p.timeout_flag = comm->timeout_flag;
        }
        return p;
      }
      static bool host_allreduce(const Exec &ex) { return ex.comm && !ex.comm->mailboxes() && ex.comm->allreduce_sum; }

      // a reduction launched earlier: the mirror slot its finaliser writes and the event the host may wait on
      struct Pending {
        Workspace *w;
        int slot;
      };
      // wait for a reduction and return the host mirror of the solver's scalar block as of that reduction
      template <typename Tr> static const double *await(const Pending &p)
      {
        cuda_ok(cudaEventSynchronize(p.w->ev[p.slot]), "event sync");
        return p.w->host + p.slot * Tr::kCount;
      }
      template <typename Tr> static void set_scalar(const Exec &ex, int idx, double v)
      {
        set_scalar_kernel<<<1, 1, 0, cs(ex.stream)>>>(workspace<Tr>(ex.stream).scalars, idx, v);
        cuda_ok(cudaGetLastError(), "scalar launch");
      }
      template <typename Tr> static void set_all(const Exec &ex, const Scalars<Tr::kCount> &s)
      {
        set_scalars_kernel<Tr::kCount><<<1, (Tr::kCount + 31) / 32 * 32, 0, cs(ex.stream)>>>(workspace<Tr>(ex.stream).scalars, s);
        cuda_ok(cudaGetLastError(), "scalar launch");
      }
      // Launch one reduction of nv sums with finaliser fin into the scalar block of Tr (kernel(T(), ra) launches it).
      // With NVLink mailboxes, or on one rank, the last block derives the scalars on the device and nothing waits.  With
      // the host all-reduce the kernel only stores its local sums; all nv of them go through the callback, the host
      // derives the scalars with the same function, writes the whole block back to the device and into the mirror slot,
      // so await() reads the same thing in both cases.  Counts the host wait in `syncs`.
      template <typename Tr, typename K>
      static Pending reduce(const Exec &ex, int nv, int fin, int &syncs, int precision, long long flops, K &&kernel)
      {
        const bool host_ar = host_allreduce(ex);
        Workspace &w = workspace<Tr>(ex.stream);
        const Pending pend {&w, (int)(w.ring++ & 7)};
        const ReduceArgs ra {w.partials, w.ticket, w.scalars, w.host_dev + pend.slot * Tr::kCount, host_ar ? (int)FIN_RAW : fin,
                             peers_of(ex.comm)};
        launch(precision, flops, [&](auto t) { kernel(t, ra); });
        cuda_ok(cudaEventRecord(w.ev[pend.slot], cs(ex.stream)), "record");
        if (host_ar) {
          Scalars<Tr::kCount> s;
          memcpy(s.s, await<Tr>(pend), sizeof(s.s));
          syncs++;
          ex.comm->allreduce_sum(s.s + Tr::kRaw, nv, ex.comm->user);
          Tr::derive(s.s, fin);
          set_all<Tr>(ex, s);
          memcpy(w.host + pend.slot * Tr::kCount, s.s, sizeof(s.s));
        }
        return pend;
      }

      template <int R> static double run(double a, const ColorSpinorField &x, double b, ColorSpinorField &y, bool write, const Exec &ex)
      {
        check_same(x, y);
        const size_t n = x.Length();
        auto axpby = [&](auto t, const ReduceArgs &ra) {
          using T = decltype(t);
          axpby_kernel<T, T, R><<<kBlocks, kThreads, 0, cs(ex.stream)>>>(a, x.data<T>(), b, y.data<T>(), n, write, ra);
        };
        if (R == R_NONE) {
          launch(x.precision, 3 * (long long)n, [&](auto t) { axpby(t, ReduceArgs {}); });
          return 0.0;
        }
        int syncs = 0; // the callers count the wait below
        return await<CgTraits>(reduce<CgTraits>(ex, 1, FIN_RAW, syncs, x.precision, 3 * (long long)n, axpby))[S_RAW0];
      }

      // Precision conversion has to go through the site/component map: the native order of fp64 fields is planes of 2
      // reals, that of fp32 fields planes of 4 (color_spinor_field_order.h FloatNOrder), so an element-wise cast
      // would permute components.  One thread per site moves its 24 reals.
      template <typename Ts, int Ns, typename Td, int Nd>
      __global__ void convert_kernel(const Ts *__restrict__ src, Td *__restrict__ dst, int volume_cb, size_t src_parity_elems,
                                     size_t dst_parity_elems)
      {
        const int x = blockIdx.x * blockDim.x + threadIdx.x;
        if (x >= volume_cb) return;
        const Ts *s = src + blockIdx.y * src_parity_elems;
        Td *d = dst + blockIdx.y * dst_parity_elems;
        double v[24];
#pragma unroll
        for (int r = 0; r < 24; r++) v[r] = s[((size_t)(r / Ns) * volume_cb + x) * Ns + r % Ns];
#pragma unroll
        for (int r = 0; r < 24; r++) d[((size_t)(r / Nd) * volume_cb + x) * Nd + r % Nd] = (Td)v[r];
      }

      void copy(ColorSpinorField &dst, const ColorSpinorField &src, const Exec &ex)
      {
        check_pair(src, dst);
        if (dst.n_parity != src.n_parity) throw Error("blas::copy: fields cover different site subsets");
        if (src.precision == dst.precision) {
          if (dst.v != src.v) cuda_ok(cudaMemcpyAsync(dst.v, src.v, src.Bytes(), cudaMemcpyDeviceToDevice, cs(ex.stream)), "copy");
          return;
        }
        const int vcb = src.VolumeCB();
        dim3 grid((vcb + 127) / 128, src.n_parity);
        const size_t se = (size_t)24 * vcb, de = (size_t)24 * vcb;
        launch(src.precision, 0, [&](auto t) {
          using Ts = decltype(t);
          using Td = std::conditional_t<sizeof(Ts) == 8, float, double>;
          convert_kernel<Ts, 16 / sizeof(Ts), Td, 16 / sizeof(Td)><<<grid, 128, 0, cs(ex.stream)>>>(src.data<Ts>(), dst.data<Td>(), vcb, se, de);
        });
      }
      void zero(ColorSpinorField &x, const Exec &ex) { cuda_ok(cudaMemsetAsync(x.v, 0, x.Bytes(), cs(ex.stream)), "memset"); }

      // gamma5 in the UKQCD basis swaps spins (0, 1) with (2, 3): the first 12 reals of a site with the last 12, which in
      // the native order (fp64: 2 reals per 16-byte plane, fp32: 4) is the first half of the planes with the second half
      __global__ void gamma5_kernel(const uint4 *__restrict__ in, uint4 *__restrict__ out, int volume_cb, int half_planes,
                                    size_t parity_elems)
      {
        const int x = blockIdx.x * blockDim.x + threadIdx.x;
        if (x >= volume_cb) return;
        const uint4 *i = in + blockIdx.y * parity_elems;
        uint4 *o = out + blockIdx.y * parity_elems;
        for (int k = 0; k < half_planes; k++) {
          const uint4 a = i[(size_t)k * volume_cb + x], b = i[(size_t)(k + half_planes) * volume_cb + x];
          o[(size_t)k * volume_cb + x] = b;
          o[(size_t)(k + half_planes) * volume_cb + x] = a;
        }
      }

      void gamma5(ColorSpinorField &out, const ColorSpinorField &in, const Exec &ex)
      {
        check_pair(in, out);
        if (out.n_parity != in.n_parity) throw Error("blas::gamma5: fields cover different site subsets");
        if (in.precision != B200_DOUBLE && in.precision != B200_SINGLE) throw Error("blas::gamma5: precision must be 8 or 4");
        const int vcb = in.VolumeCB(), planes = 24 * in.precision / 16;
        gamma5_kernel<<<dim3((vcb + 127) / 128, in.n_parity), 128, 0, cs(ex.stream)>>>(
          static_cast<const uint4 *>(in.v), static_cast<uint4 *>(out.v), vcb, planes / 2, (size_t)planes * vcb);
        cuda_ok(cudaGetLastError(), "gamma5 launch");
      }
      void axpy(double a, const ColorSpinorField &x, ColorSpinorField &y, const Exec &ex) { run<R_NONE>(a, x, 1.0, y, true, ex); }
      double norm2(const ColorSpinorField &x, const Exec &ex)
      {
        return run<R_NORM_Y>(0.0, x, 1.0, const_cast<ColorSpinorField &>(x), false, ex);
      }
      double axpyNorm(double a, const ColorSpinorField &x, ColorSpinorField &y, const Exec &ex) { return run<R_NORM_Y>(a, x, 1.0, y, true, ex); }

      // ---- CG iteration pieces (used by invertCG below)
      // <p, Ap> -> pAp, alpha = r2 / pAp (device)
      static Pending cg_dot(const ColorSpinorField &p, const ColorSpinorField &Ap, const Exec &ex, int &syncs)
      {
        check_same(p, Ap);
        const size_t n = p.Length();
        return reduce<CgTraits>(ex, 1, FIN_PAP, syncs, p.precision, 2 * (long long)n, [&](auto t, const ReduceArgs &ra) {
          using T = decltype(t);
          axpby_kernel<T, T, R_DOT_XY><<<kBlocks, kThreads, 0, cs(ex.stream)>>>(0.0, p.data<T>(), 1.0, Ap.data<T>(), n, false, ra);
        });
      }
      static Pending cg_update_r(ColorSpinorField &r, const ColorSpinorField &Ap, const Exec &ex, int &syncs)
      {
        check_same(r, Ap);
        const size_t n = r.Length();
        return reduce<CgTraits>(ex, 1, FIN_R2, syncs, r.precision, 4 * (long long)n, [&](auto t, const ReduceArgs &ra) {
          using T = decltype(t);
          cg_update_r_kernel<T><<<kBlocks, kThreads, 0, cs(ex.stream)>>>(r.data<T>(), Ap.data<T>(), n, ra);
        });
      }
      static void cg_update_xp(ColorSpinorField &x, ColorSpinorField &p, const ColorSpinorField &r, const Exec &ex)
      {
        check_same(x, p);
        const size_t n = p.Length();
        const double *S = workspace<CgTraits>(ex.stream).scalars;
        launch(p.precision, 4 * (long long)n, [&](auto t) {
          using T = decltype(t);
          cg_update_xp_kernel<T><<<kBlocks, kThreads, 0, cs(ex.stream)>>>(x.data<T>(), p.data<T>(), r.data<T>(), n, S);
        });
      }
      static void cg_replace_r(ColorSpinorField &p, ColorSpinorField &r, const ColorSpinorField &r_new, const Exec &ex)
      {
        check_same(p, r_new);
        const size_t n = p.Length();
        launch(p.precision, 2 * (long long)n, [&](auto t) {
          using T = decltype(t);
          cg_replace_r_kernel<T><<<kBlocks, kThreads, 0, cs(ex.stream)>>>(p.data<T>(), r.data<T>(), r_new.data<T>(), n);
        });
      }

      // ---- BiCGStab iteration pieces (used by invertBiCGStab below); all operands share the sloppy precision
      // <a, b> (K1 with BF_ALPHA; rho = <r0, r> with BF_RHO)
      static Pending bicg_cdot(const ColorSpinorField &a, const ColorSpinorField &b, int fin, const Exec &ex, int &syncs)
      {
        check_same(a, b);
        const size_t n = a.Length() / 2;
        return reduce<BicgTraits>(ex, 2, fin, syncs, a.precision, 8 * (long long)n, [&](auto t, const ReduceArgs &ra) {
          using T = decltype(t);
          bicg_cdot_kernel<T><<<kBlocks, kThreads, 0, cs(ex.stream)>>>(a.data<T>(), b.data<T>(), n, ra);
        });
      }
      // K2
      static void bicg_update_s(ColorSpinorField &r, const ColorSpinorField &v, const Exec &ex)
      {
        check_same(r, v);
        const size_t n = r.Length() / 2;
        const double *S = workspace<BicgTraits>(ex.stream).scalars;
        launch(r.precision, 8 * (long long)n, [&](auto t) {
          using T = decltype(t);
          bicg_update_s_kernel<T><<<kBlocks, kThreads, 0, cs(ex.stream)>>>(r.data<T>(), v.data<T>(), n, S);
        });
      }
      // K3
      static Pending bicg_ts(const ColorSpinorField &t, const ColorSpinorField &s, const Exec &ex, int &syncs)
      {
        check_same(t, s);
        const size_t n = t.Length() / 2;
        return reduce<BicgTraits>(ex, 4, BF_OMEGA, syncs, t.precision, 16 * (long long)n, [&](auto z, const ReduceArgs &ra) {
          using T = decltype(z);
          bicg_ts_kernel<T><<<kBlocks, kThreads, 0, cs(ex.stream)>>>(t.data<T>(), s.data<T>(), n, ra);
        });
      }
      // K4
      static Pending bicg_update_xr(ColorSpinorField &x, ColorSpinorField &r, const ColorSpinorField &p, const ColorSpinorField &t,
                                    const ColorSpinorField &r0, const Exec &ex, int &syncs)
      {
        check_same(x, r, p, t, r0);
        const size_t n = x.Length() / 2;
        return reduce<BicgTraits>(ex, 3, BF_BETA, syncs, x.precision, 36 * (long long)n, [&](auto z, const ReduceArgs &ra) {
          using T = decltype(z);
          bicg_update_xr_kernel<T><<<kBlocks, kThreads, 0, cs(ex.stream)>>>(x.data<T>(), r.data<T>(), p.data<T>(), t.data<T>(),
                                                                            r0.data<T>(), n, ra);
        });
      }
      // K5
      static void bicg_update_p(ColorSpinorField &p, const ColorSpinorField &r, const ColorSpinorField &v, const Exec &ex)
      {
        check_same(p, r, v);
        const size_t n = p.Length() / 2;
        const double *S = workspace<BicgTraits>(ex.stream).scalars;
        launch(p.precision, 16 * (long long)n, [&](auto t) {
          using T = decltype(t);
          bicg_update_p_kernel<T><<<kBlocks, kThreads, 0, cs(ex.stream)>>>(p.data<T>(), r.data<T>(), v.data<T>(), n, S);
        });
      }

      // ---- multi-shift CG iteration pieces (used by invertMultiShiftCG below); all operands share the sloppy precision
      template <typename T> static const Vec<T> *vec(const ColorSpinorField &f) { return reinterpret_cast<const Vec<T> *>(f.v); }
      template <typename T> static Vec<T> *vec(ColorSpinorField &f) { return reinterpret_cast<Vec<T> *>(f.v); }
      template <typename... F> static size_t ms_check(const ColorSpinorField &x, const F &...ys)
      {
        check_same(x, ys...);
        for (const ColorSpinorField *f : {&x, &ys...})
          if (reinterpret_cast<uintptr_t>(f->v) % 16) throw Error("multi-shift CG: fields must be 16-byte aligned");
        return x.Length(); // a multiple of 24 reals, so of every vector width
      }
      template <typename T> static MsFields<T> ms_fields(const std::vector<ColorSpinorField> &x, const std::vector<ColorSpinorField> &p)
      {
        MsFields<T> f {};
        for (size_t j = 0; j < p.size(); j++) {
          if (j < x.size()) f.x[j] = x[j].data<T>();
          f.p[j] = p[j].data<T>();
        }
        return f;
      }
      static Pending ms_dot(const ColorSpinorField &p, ColorSpinorField &Ap, double sigma, const Exec &ex, int &syncs)
      {
        const size_t n = ms_check(p, Ap);
        return reduce<MsTraits>(ex, 1, FIN_PAP, syncs, p.precision, 4 * (long long)n, [&](auto t, const ReduceArgs &ra) {
          using T = decltype(t);
          ms_dot_kernel<T><<<kBlocks, kThreads, 0, cs(ex.stream)>>>(vec<T>(p), vec<T>(Ap), sigma, n / Vec<T>::W, ra);
        });
      }
      static Pending ms_update_r(ColorSpinorField &r, const ColorSpinorField &Ap, const Exec &ex, int &syncs)
      {
        const size_t n = ms_check(r, Ap);
        return reduce<MsTraits>(ex, 1, FIN_R2, syncs, r.precision, 4 * (long long)n, [&](auto t, const ReduceArgs &ra) {
          using T = decltype(t);
          ms_update_r_kernel<T><<<kBlocks, kThreads, 0, cs(ex.stream)>>>(vec<T>(r), vec<T>(Ap), n / Vec<T>::W, ra);
        });
      }
      // n_active: the host's view of the active shifts, for the flop count only (the kernel reads M_NUPD)
      static void ms_update_xp(const std::vector<ColorSpinorField> &x, const std::vector<ColorSpinorField> &p, const ColorSpinorField &r,
                               int n_active, const Exec &ex)
      {
        size_t n = 0;
        for (size_t j = 0; j < p.size(); j++) n = ms_check(r, x[j], p[j]);
        const double *S = workspace<MsTraits>(ex.stream).scalars;
        launch(r.precision, 5 * (long long)n * n_active, [&](auto t) {
          using T = decltype(t);
          ms_update_xp_kernel<T><<<kBlocks, kThreads, 0, cs(ex.stream)>>>(ms_fields<T>(x, p), vec<T>(r), n / Vec<T>::W, S);
        });
      }
      static void ms_replace_r(const std::vector<ColorSpinorField> &p, ColorSpinorField &r, const ColorSpinorField &r_new, double r2,
                               const Exec &ex)
      {
        size_t n = 0;
        for (const ColorSpinorField &f : p) n = ms_check(r, f, r_new);
        double *S = workspace<MsTraits>(ex.stream).scalars;
        launch(r.precision, 3 * (long long)n * p.size(), [&](auto t) {
          using T = decltype(t);
          ms_replace_r_kernel<T><<<kBlocks, kThreads, 0, cs(ex.stream)>>>(ms_fields<T>({}, p), vec<T>(r), vec<T>(r_new), n / Vec<T>::W, S, r2);
        });
      }
      // the device scalar block of Tr as it stands once the stream has drained
      template <typename Tr> static std::vector<double> fetch(const Exec &ex)
      {
        std::vector<double> S(Tr::kCount);
        cuda_ok(cudaMemcpyAsync(S.data(), workspace<Tr>(ex.stream).scalars, sizeof(double) * Tr::kCount, cudaMemcpyDeviceToHost,
                                cs(ex.stream)), "memcpy(scalars)");
        cuda_ok(cudaStreamSynchronize(cs(ex.stream)), "sync");
        return S;
      }
    } // namespace blas

    // ------------------------------------------------------------------ the even-odd operator
    Dirac::Dirac(SiteTerm term_, bool schur_, const DiracParam &p) :
      gauge(p.gauge), clover(p.clover), kappa(p.kappa), mu(p.mu), matpcType(p.matpcType), dagger(p.dagger), comm(p.comm),
      stream(p.stream), term(term_), schur(schur_)
    {
      if (!gauge) throw Error("operator needs a gauge field");
      if (term == SiteTerm::Clover) {
        if (!clover) throw Error("clover operator needs a clover field");
        if (schur && !clover->has_inverse() && !clover->c.dynamic_inverse)
          throw Error("even-odd preconditioned clover operator needs A^-1 (a static inverse field or dynamic_inverse)");
      }
      for (int d = 0; d < 4; d++) commDim[d] = p.commDim[d];
      symmetric = (matpcType == QUDA_MATPC_EVEN_EVEN || matpcType == QUDA_MATPC_ODD_ODD);
      this_parity = (matpcType == QUDA_MATPC_EVEN_EVEN || matpcType == QUDA_MATPC_EVEN_EVEN_ASYMMETRIC) ? 0 : 1;
      other_parity = 1 - this_parity;
    }

    Dirac *Dirac::create(const std::string &type, const DiracParam &p)
    {
      if (type == "wilson") return new Dirac(SiteTerm::Identity, false, p);
      if (type == "wilsonpc") return new Dirac(SiteTerm::Identity, true, p);
      if (type == "clover") return new Dirac(SiteTerm::Clover, false, p);
      if (type == "cloverpc") return new Dirac(SiteTerm::Clover, true, p);
      if (type == "twistedmass") return new Dirac(SiteTerm::Twist, false, p);
      if (type == "twistedmasspc") return new Dirac(SiteTerm::Twist, true, p);
      throw Error("no operator of type '" + type + "' in this engine");
    }

    static void need_single_parity(const ColorSpinorField &a, const ColorSpinorField &b)
    {
      if (a.n_parity != 1 || b.n_parity != 1) throw Error("this operation acts on single-parity fields");
      if (a.v == b.v) throw Error("input and output must be different fields");
    }
    static void need_full(const ColorSpinorField &a, const ColorSpinorField &b)
    {
      if (a.n_parity != 2 || b.n_parity != 2) throw Error("this operation acts on full (two-parity) fields");
    }

    // One Dslash launch: out = [x +] k * (site-term fused in the epilogue) D in
    //   Fuse::None     : out = D in                | x + k D in
    //   Fuse::A        : out = A x + k D in        (always with x)
    //   Fuse::AinvPost : out = A^-1 D in           | x + k A^-1 D in
    // For the identity site term all three coincide with the Wilson form.
    void Dirac::hop(ColorSpinorField &out, const ColorSpinorField &in, int parity, Fuse f, const ColorSpinorField *x, double k) const
    {
      need_single_parity(in, out);
      if (x && k == 0.0) {
        // x + 0 D in: the launch ABI reads a == 0 as "no x term", so the hop is skipped rather than issued (kappa = 0)
        if (f == Fuse::A) site(out, *x, parity, false);
        else blas::copy(out, *x, exec());
        return;
      }
      const ColorSpinorField &xf = x ? *x : in;
      const double a = x ? k : 0.0;
      if (term == SiteTerm::Identity || f == Fuse::None) {
        ApplyWilson(out, in, *gauge, a, xf, parity, dagger, commDim, comm, stream);
      } else if (term == SiteTerm::Clover) {
        if (f == Fuse::A) {
          if (!x) throw Error("A x + k D in needs x");
          ApplyWilsonClover(out, in, *gauge, *clover, a, xf, parity, dagger, commDim, comm, stream);
        } else {
          ApplyWilsonCloverPreconditioned(out, in, *gauge, *clover, a, xf, parity, dagger, commDim, comm, stream);
        }
      } else { // twist: A = 1 + i 2 kappa mu gamma5, A^-1 = (1 - i 2 kappa mu gamma5) / (1 + (2 kappa mu)^2)
        if (f == Fuse::A) {
          if (!x) throw Error("the twisted-mass Dslash exists only in its xpay form");
          ApplyTwistedMass(out, in, *gauge, a, 2 * mu * kappa, xf, parity, dagger, commDim, comm, stream);
        } else {
          const double tw = -2.0 * kappa * mu;
          const double nrm = 1.0 / (1.0 + tw * tw);
          const bool asym = !symmetric && dagger;
          ApplyTwistedMassPreconditioned(out, in, *gauge, x ? k * nrm : nrm, tw, x != nullptr, xf, parity, dagger, asym, commDim, comm, stream);
        }
      }
      dslash_applications++;
    }

    // out = A in or A^-1 in on one parity
    void Dirac::site(ColorSpinorField &out, const ColorSpinorField &in, int parity, bool inverse) const
    {
      switch (term) {
      case SiteTerm::Identity: blas::copy(out, in, exec()); break;
      case SiteTerm::Clover: ApplyClover(out, in, *clover, inverse, parity, stream); break;
      case SiteTerm::Twist: ApplyTwistGamma(out, in, kappa, mu, dagger, inverse, stream); break;
      }
    }

    void Dirac::Dslash(ColorSpinorField &out, const ColorSpinorField &in, int parity) const
    {
      if (term == SiteTerm::Twist && !schur) throw Error("the unpreconditioned twisted-mass Dslash exists only in its xpay form");
      hop(out, in, parity, schur ? Fuse::AinvPost : Fuse::None, nullptr, 0.0);
    }

    void Dirac::DslashXpay(ColorSpinorField &out, const ColorSpinorField &in, int parity, const ColorSpinorField &x, double k) const
    {
      hop(out, in, parity, schur ? Fuse::AinvPost : Fuse::A, &x, k);
    }

    void Dirac::M(ColorSpinorField &out, const ColorSpinorField &in) const
    {
      if (!schur) {
        // out_p = A_p in_p - kappa D in_{1-p}
        need_full(out, in);
        const bool one_launch = term != SiteTerm::Twist && !(comm && comm->partitioned()) && kappa != 0.0;
        if (one_launch) { // both parities in one launch (full-field kernel)
          if (term == SiteTerm::Identity)
            ApplyWilson(out, in, *gauge, -kappa, in, QUDA_INVALID_PARITY, dagger, commDim, comm, stream);
          else
            ApplyWilsonClover(out, in, *gauge, *clover, -kappa, in, QUDA_INVALID_PARITY, dagger, commDim, comm, stream);
          dslash_applications += 2;
        } else {
          for (int p = 0; p < 2; p++) {
            auto o = out.parity_view(p);
            const auto x = in.parity_view(p);
            hop(o, in.parity_view(1 - p), p, Fuse::A, &x, -kappa);
          }
        }
        return;
      }
      // Schur complement on `this_parity`
      const double k2 = -kappa * kappa;
      Scratch tmp(stream, in, 1);
      if (term == SiteTerm::Clover && symmetric && dagger) {
        // (1 - k^2 A^-1 D A^-1 D)^dagger = 1 - k^2 D^dagger A^-1 D^dagger A^-1   (A hermitian)
        site(out, in, this_parity, true);
        hop(tmp, out, other_parity, Fuse::AinvPost, nullptr, 0.0);
        hop(out, tmp, this_parity, Fuse::None, &in, k2);
      } else {
        hop(tmp, in, other_parity, Fuse::AinvPost, nullptr, 0.0);
        hop(out, tmp, this_parity, symmetric ? Fuse::AinvPost : Fuse::A, &in, k2);
      }
    }

    void Dirac::Mdag(ColorSpinorField &out, const ColorSpinorField &in) const
    {
      flipDagger();
      try {
        M(out, in);
      } catch (...) {
        flipDagger();
        throw;
      }
      flipDagger();
    }

    void Dirac::MdagM(ColorSpinorField &out, const ColorSpinorField &in) const
    {
      Scratch tmp(stream, in, in.n_parity);
      M(tmp, in);
      Mdag(out, tmp);
    }

    // Full-system solve through the Schur complement: M x = b  <=>  M_pc x_e = src, x_o from x_e.
    //   symmetric : src = A_e^-1 (b_e + k D_eo A_o^-1 b_o)       asymmetric : src = b_e + k D_eo A_o^-1 b_o
    // The preconditioned source is built in the other-parity half of x, the solution lives in the this-parity half.
    void Dirac::prepare(ColorSpinorField &sol, ColorSpinorField &src, ColorSpinorField &x, const ColorSpinorField &b,
                        QudaSolutionType st) const
    {
      const bool pc_solution = (st == QUDA_MATPC_SOLUTION || st == QUDA_MATPCDAG_MATPC_SOLUTION);
      if (!schur) {
        if (pc_solution) throw Error("a preconditioned solution type needs an even-odd preconditioned operator");
        src = b;
        sol = x;
        return;
      }
      if (pc_solution) {
        src = b;
        sol = x;
        return;
      }
      need_full(x, b);
      src = x.parity_view(other_parity);
      sol = x.parity_view(this_parity);
      const auto b_this = b.parity_view(this_parity), b_other = b.parity_view(other_parity);
      if (term == SiteTerm::Identity) {
        hop(src, b_other, this_parity, Fuse::None, &b_this, kappa);
        return;
      }
      Scratch tmp(stream, b, 1);
      if (symmetric) {
        site(src, b_other, other_parity, true);
        hop(tmp, src, this_parity, Fuse::None, &b_this, kappa);
        site(src, tmp, this_parity, true);
      } else {
        site(tmp, b_other, other_parity, true);
        hop(src, tmp, this_parity, Fuse::None, &b_this, kappa);
      }
    }

    // ---- clover force (lib/clover_force.cpp)
    void computeCloverForce(void *mom, double dt, const std::vector<ColorSpinorField> &x, const double *coeff, double kappa2,
                            double ck, double multiplicity, const void *const qdp[4], const void *packed, const Dirac &op)
    {
      if (!op.is_clover() || !op.pc()) throw Error("the clover force needs an even-odd preconditioned clover operator");
      if (op.is_symmetric()) throw Error("the clover force needs asymmetric preconditioning (EVEN_EVEN_ASYMMETRIC or ODD_ODD_ASYMMETRIC)");
      if (op.Comm() && op.Comm()->partitioned()) throw Error("the clover force runs on one GPU: the lattice must not be partitioned");
      const int n = (int)x.size();
      if (n < 1 || n > B200_MAX_SHIFTS) throw Error("the clover force takes 1 to " + std::to_string(B200_MAX_SHIFTS) + " solutions");
      for (const auto &f : x)
        if (f.n_parity != 1 || f.precision != op.Precision()) throw Error("each solution must be a single-parity field of the operator's precision");
      const int par = op.thisParity(), oth = 1 - par;
      const Exec ex = op.exec();
      // p_i and the other parity of x_i, prepared along the dagger branch of the reference (gamma5, dagger Dslash of the
      // other parity, Mhat^+, gamma5; then the plain Dslash): for solutions of (Mhat^+ Mhat + sigma) x = phi this is the
      // derivative of phi^+ (Mhat^+ Mhat + sigma)^-1 phi.  That branch hands p to the outer products in x's place.
      std::vector<std::unique_ptr<Scratch>> xf, pf;
      std::vector<const void *> xp, pp;
      Scratch t(op.Stream(), x[0], 1);
      for (int i = 0; i < n; i++) {
        xf.emplace_back(new Scratch(op.Stream(), x[i], 2));
        pf.emplace_back(new Scratch(op.Stream(), x[i], 2));
        ColorSpinorField &X = *xf.back(), &P = *pf.back();
        auto x_oth = X.parity_view(oth), x_par = X.parity_view(par), p_par = P.parity_view(par), p_oth = P.parity_view(oth);
        blas::gamma5(t, x[i], ex);
        op.flipDagger();
        try {
          op.Dslash(x_oth, t, oth);
          op.M(p_par, t);
        } catch (...) {
          op.flipDagger();
          throw;
        }
        op.flipDagger();
        blas::gamma5(x_oth, x_oth, ex);
        op.Dslash(p_oth, p_par, oth);
        blas::gamma5(P, P, ex);
        blas::copy(x_par, x[i], ex);
        xp.push_back(P.v);
        pp.push_back(X.v);
      }
      std::vector<double> fc(n), eps(2 * (size_t)n);
      for (int i = 0; i < n; i++) {
        fc[i] = 2.0 * dt * coeff[i] * kappa2;
        // the reference indexes epsilon by site parity; its first entry belongs to the matpc parity
        eps[2 * i + par] = 2.0 * ck * coeff[i] * dt;
        eps[2 * i + oth] = -kappa2 * 2.0 * ck * coeff[i] * dt;
      }
      const GaugeField &U = op.Gauge();
      abi_ok(b200_clover_force_accumulate(mom, qdp, packed, U.X, op.Precision(), n, xp.data(), pp.data(), fc.data(), eps.data(),
                                          2.0 * ck * multiplicity * dt, oth, op.Stream()));
      cuda_ok(cudaStreamSynchronize(cs(op.Stream())), "clover force");
    }

    // x_o = A_o^-1 (b_o + k D_oe x_e)
    void Dirac::reconstruct(ColorSpinorField &x, const ColorSpinorField &b, QudaSolutionType st) const
    {
      if (!schur || st == QUDA_MATPC_SOLUTION || st == QUDA_MATPCDAG_MATPC_SOLUTION) return;
      need_full(x, b);
      auto x_other = x.parity_view(other_parity);
      const auto x_this = x.parity_view(this_parity), b_other = b.parity_view(other_parity);
      if (term == SiteTerm::Identity) {
        hop(x_other, x_this, other_parity, Fuse::None, &b_other, kappa);
        return;
      }
      Scratch tmp(stream, b, 1);
      hop(tmp, x_this, other_parity, Fuse::None, &b_other, kappa);
      site(x_other, tmp, other_parity, true);
    }

    // ------------------------------------------------------------------ what the solvers share
    // Argument checks, the precise work fields r (residual), y (accumulated solution) and tmp, the sloppy solution xS and
    // residual rS (r itself when both operators have one precision), the true residual in the precise operator `op`
    // (MdagM for CG and multi-shift CG, M for BiCGStab) plus `shift`, and the statistics of SolverParam.
    namespace
    {
      struct Solve {
        using Op = void (Dirac::*)(ColorSpinorField &, const ColorSpinorField &) const;
        const Dirac &mat, &matSloppy;
        const Op op;
        ColorSpinorField &x;
        const ColorSpinorField &b;
        const Exec ex;
        const std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
        const long long flops0, ds0;
        const int sp;
        const bool same_prec, host_ar;
        int syncs = 0;
        int k = 0;         // iterations run
        bool done = false; // set by the solver's decision
        Scratch r_s, y_s, tmp_s, xS_s;
        std::unique_ptr<Scratch> rS_s;
        ColorSpinorField &r = r_s.f, &y = y_s.f, &tmp = tmp_s.f, &xS = xS_s.f;
        ColorSpinorField rS;
        double b2 = 0.0;
        double shift = 0.0; // residual() is taken for op + shift (multi-shift CG; 0 for CG and BiCGStab)

        // checks the arguments; returns the sloppy precision
        static int sloppy_precision(const Dirac &mat, const Dirac &matSloppy, const ColorSpinorField &x, const ColorSpinorField &b)
        {
          if (matSloppy.Stream() != mat.Stream()) throw Error("precise and sloppy operators must share a stream");
          const int sp = matSloppy.Precision();
          if (x.precision != mat.Precision() || b.precision != mat.Precision()) throw Error("x and b must have the precise operator's precision");
          if (sp != 8 && sp != 4) throw Error("the sloppy operator must be double or single precision");
          if (&mat != &matSloppy && sp > x.precision) throw Error("the sloppy operator is more precise than the precise one");
          return sp;
        }
        Solve(const Dirac &mat_, const Dirac &matSloppy_, Op op_, ColorSpinorField &x_, const ColorSpinorField &b_) :
          mat(mat_), matSloppy(matSloppy_), op(op_), x(x_), b(b_), ex(mat_.exec()), flops0(blas::flops()),
          ds0(mat_.DslashApplications() + matSloppy_.DslashApplications()), sp(sloppy_precision(mat_, matSloppy_, x_, b_)),
          same_prec(sp == x_.precision), host_ar(blas::host_allreduce(ex)), r_s(ex.stream, x.X, x.precision, x.n_parity),
          y_s(ex.stream, x.X, x.precision, x.n_parity), tmp_s(ex.stream, x.X, x.precision, x.n_parity), xS_s(sloppy())
        {
          // work fields come from the per-stream scratch pool: a second solve on the same stream allocates nothing
          if (!same_prec) rS_s.reset(new Scratch(sloppy()));
          rS = same_prec ? r : rS_s->f;
        }
        Scratch sloppy() const { return Scratch(ex.stream, x.X, sp, x.n_parity); }

        // b2 = |b|^2; if b == 0, x = 0 and there is nothing to solve
        bool zero_source()
        {
          b2 = blas::norm2(b, ex);
          syncs++;
          if (b2 != 0.0) return false;
          blas::zero(x, ex);
          return true;
        }
        bool zero_source(SolverParam &param)
        {
          if (!zero_source()) return false;
          param.iter = 0;
          param.true_res = 0.0;
          return true;
        }
        // r = b - op z in the precise operator; returns |r|^2
        double residual(const ColorSpinorField &z)
        {
          (mat.*op)(tmp, z);
          if (shift != 0.0) blas::axpy(shift, z, tmp, ex);
          blas::copy(r, b, ex);
          const double r2 = blas::axpyNorm(-1.0, tmp, r, ex);
          syncs++;
          return r2;
        }
        // y = x, r = b - op x, rS = r, xS = 0; returns |r|^2
        double start()
        {
          blas::copy(y, x, ex);
          const double r2 = residual(x);
          if (!same_prec) blas::copy(rS, r, ex);
          blas::zero(xS, ex);
          return r2;
        }
        // acc += sloppy, staged through tmp when the precisions differ
        void fold(ColorSpinorField &acc, const ColorSpinorField &sloppy)
        {
          if (same_prec) {
            blas::axpy(1.0, sloppy, acc, ex);
          } else {
            blas::copy(tmp, sloppy, ex);
            blas::axpy(1.0, tmp, acc, ex);
          }
        }
        void fold() { fold(y, xS); }
        // reliable update: fold the sloppy solution into y, xS = 0, r = b - op y; returns |r|^2
        double reliable_update()
        {
          fold();
          blas::zero(xS, ex);
          return residual(y);
        }
        // The iteration loop of every solver.  step() queues one iteration and returns the reduction whose scalar block
        // (of Tr) the host decides on; decide(S, j) reads that block as of iteration j and returns true if it replaced
        // the residual.  No iteration waits for the host: while the GPU runs iteration k the host decides on k - 1.  With
        // the host-callback all-reduce every reduction has already been waited for, so it decides on k at once.
        template <typename Tr, typename Step, typename Decide> void iterate(int maxiter, Step &&step, Decide &&decide)
        {
          blas::Pending prev {};
          bool have_prev = false;
          while (!done && k < maxiter) {
            const blas::Pending pend = step();
            k++;
            if (host_ar) {
              decide(blas::await<Tr>(pend), k);
              continue;
            }
            bool replaced = false;
            if (have_prev) {
              replaced = decide(blas::await<Tr>(prev), k - 1);
              syncs++;
            }
            // after a replacement the pending scalars belong to the recursion before it
            have_prev = !replaced;
            prev = pend;
          }
        }
        // x = y + xS, its true residual, and the statistics
        void finish(SolverParam &param)
        {
          fold();
          blas::copy(x, y, ex);
          const double tr2 = residual(x);
          complete(param);
          param.iter = k;
          param.true_res = std::sqrt(tr2 / b2);
        }
        // waits for the solve, checks the halo exchange and fills in the statistics common to every solver
        template <typename P> void complete(P &param)
        {
          cuda_ok(cudaStreamSynchronize(cs(ex.stream)), "sync");
          if (halo_timed_out(ex.comm, ex.stream)) throw Error("a halo wait timed out during the solve: the result is not valid");
          param.host_syncs = syncs;
          param.secs = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
          const long long nds = mat.DslashApplications() + matSloppy.DslashApplications() - ds0;
          const double fl = (double)(blas::flops() - flops0) + (double)nds * 1320.0 * x.VolumeCB();
          param.gflops = fl / param.secs * 1e-9;
        }
      };

      // The reliable-update rule of the reference's CG (lib/inv_cg_quda.cpp), shared by CG and multi-shift CG: |r| is
      // measured against its value r0Norm after the last update and against its maxima since then.
      struct CgReliable {
        double r0Norm, maxrx, maxrr;
        explicit CgReliable(double r2) { reset(r2); }
        // tracks the maxima; true if |r|^2 = r2 calls for an update (in mixed precision always once converged)
        bool update(double r2, double delta, bool mixed, bool converged)
        {
          const double rNorm = std::sqrt(r2);
          if (rNorm > maxrx) maxrx = rNorm;
          if (rNorm > maxrr) maxrr = rNorm;
          return mixed && ((rNorm < delta * maxrx && r0Norm <= maxrx) || (rNorm < delta * r0Norm && r0Norm <= maxrr) || converged);
        }
        // after an update that left |r|^2 = r2
        void reset(double r2) { r0Norm = maxrx = maxrr = std::sqrt(r2); }
      };
    } // namespace

    // ------------------------------------------------------------------ CG (normal equations) with reliable updates
    // Same recurrences and reliable-update criterion as the reference's CG (lib/inv_cg_quda.cpp:237-420), restructured so
    // that no iteration waits for the host: pAp, r2, alpha, beta live on the device (written by the reduction
    // finalisers, read by the next update kernel); the host reads r2 of iteration k-1 while the GPU runs iteration k and
    // takes its convergence / reliable-update decisions one iteration late.  A late reliable update repairs the search
    // direction with p += r_true - r_sloppy, which restores p = r_true + beta p_old exactly.
    void invertCG(const Dirac &mat, const Dirac &matSloppy, ColorSpinorField &x, const ColorSpinorField &b, SolverParam &param)
    {
      using namespace blas;
      Solve s(mat, matSloppy, &Dirac::MdagM, x, b);
      const Exec &ex = s.ex;
      Scratch p_s = s.sloppy(), Ap_s = s.sloppy();
      ColorSpinorField &p = p_s.f, &Ap = Ap_s.f, &rS = s.rS;
      if (s.zero_source(param)) return;

      double r2 = s.start();
      copy(p, rS, ex);
      set_scalar<CgTraits>(ex, S_R2, r2);
      const double stop = param.tol * param.tol * s.b2;
      CgReliable rel(r2);
      param.reliable_updates = 0;

      // convergence / reliable-update decision on the scalar block after an iteration (CG has no done flag, so the
      // iteration queued behind it runs and counts); true if the recursion was restarted
      auto decide = [&](const double *S, int) {
        const bool converged = S[S_R2] <= stop;
        if (!rel.update(S[S_R2], param.delta, !s.same_prec, converged)) {
          s.done = converged;
          return false;
        }
        // the true residual repairs the recursion: p += r_true - rS ; rS = r_true
        r2 = s.reliable_update();
        copy(Ap, s.r, ex); // the true residual in the sloppy precision; Ap is free until the next iteration
        cg_replace_r(p, rS, Ap, ex);
        set_scalar<CgTraits>(ex, S_R2, r2);
        param.reliable_updates++;
        rel.reset(r2);
        s.done = r2 <= stop;
        return true;
      };
      s.iterate<CgTraits>(param.maxiter, [&] {
        matSloppy.MdagM(Ap, p);
        cg_dot(p, Ap, ex, s.syncs);
        const Pending pr = cg_update_r(rS, Ap, ex, s.syncs);
        cg_update_xp(s.xS, p, rS, ex);
        return pr;
      }, decide);
      s.finish(param);
    }

    // ------------------------------------------------------------------ BiCGStab (M x = b) with reliable updates
    // The reference's recurrence and reliable-update criterion (lib/inv_bicgstab_quda.cpp:71-80, 187-355) with CG's
    // structure: rho, alpha, omega, beta and |r|^2 live on the device (blas::bicg_scalars, run by the reduction finalisers),
    // one iteration is v = M p, K1..K5 and t = M s around them, and the host reads |r|^2 and the breakdown word of
    // iteration k - 1 while the GPU runs iteration k.  When |r|^2 reaches the stopping value the K4 finaliser sets B_DONE
    // and the kernels of the iteration already queued behind it return at once, so the solution is that of the iteration
    // the host reports.
    // A late reliable update replaces r (and rho = <r0, r>) after iteration k has run and keeps p.  The recursion stays
    // consistent because x and r are only ever changed together, x += alpha p + omega s against r -= alpha M p + omega M s,
    // so r = b - M x holds for any search direction p; keeping p only perturbs the bi-orthogonality of the directions by
    // the drift r_true - r_sloppy, and rho is recomputed so that alpha = rho / <r0, M p> and the next beta refer to the
    // residual the recursion now carries.  A restart after a breakdown additionally sets r0 = p = r.
    void invertBiCGStab(const Dirac &mat, const Dirac &matSloppy, ColorSpinorField &x, const ColorSpinorField &b, SolverParam &param)
    {
      using namespace blas;
      Solve s(mat, matSloppy, &Dirac::M, x, b);
      const Exec &ex = s.ex;
      Scratch p_s = s.sloppy(), v_s = s.sloppy(), t_s = s.sloppy(), r0_s = s.sloppy();
      ColorSpinorField &p = p_s.f, &v = v_s.f, &t = t_s.f, &r0 = r0_s.f;
      ColorSpinorField &rS = s.rS; // sloppy residual; holds s between K2 and K4
      if (s.zero_source(param)) return;
      const double stop = param.tol * param.tol * s.b2;
      double r2 = 0.0, maxrr = 0.0;
      param.reliable_updates = 0;

      // reliable update in the precise operator, then rS = r; clears the device flags
      auto true_residual = [&]() {
        r2 = s.reliable_update();
        if (!s.same_prec) copy(rS, s.r, ex);
        set_scalar<BicgTraits>(ex, B_R2, r2);
        set_scalar<BicgTraits>(ex, B_DONE, 0.0);
        set_scalar<BicgTraits>(ex, B_BREAK, 0.0);
        maxrr = std::sqrt(r2);
      };
      auto recompute_rho = [&]() { bicg_cdot(r0, rS, BF_RHO, ex, s.syncs); };

      // r = b - M x, r0 = p = r, rho = <r0, r>
      r2 = s.start();
      maxrr = std::sqrt(r2);
      copy(r0, rS, ex);
      copy(p, rS, ex);
      Scalars<B_COUNT> s0 {};
      s0.s[B_R2] = r2;
      s0.s[B_STOP] = stop;
      set_all<BicgTraits>(ex, s0);
      recompute_rho();
      s.done = r2 <= stop;

      // convergence / reliable-update / restart decision on the scalar block after iteration j; true if r was replaced
      auto decide = [&](const double *S, int j) {
        r2 = S[B_R2];
        const bool converged = S[B_DONE] != 0.0, broke = S[B_BREAK] != 0.0;
        if (converged) s.k = j; // the iteration queued after j returned at once
        const double rNorm = std::sqrt(r2);
        if (rNorm > maxrr) maxrr = rNorm;
        if (broke) { // restart from the true residual with a new shadow residual
          true_residual();
          copy(r0, rS, ex);
          copy(p, rS, ex);
        } else if (!s.same_prec && (converged || rNorm < param.delta * maxrr)) {
          true_residual(); // reliable update: p is kept
        } else {
          s.done = converged;
          return false;
        }
        recompute_rho();
        param.reliable_updates++;
        s.done = r2 <= stop;
        return true;
      };
      s.iterate<BicgTraits>(param.maxiter, [&] {
        matSloppy.M(v, p);
        bicg_cdot(r0, v, BF_ALPHA, ex, s.syncs);                            // K1
        bicg_update_s(rS, v, ex);                                            // K2
        matSloppy.M(t, rS);
        bicg_ts(t, rS, ex, s.syncs);                                         // K3
        const Pending p4 = bicg_update_xr(s.xS, rS, p, t, r0, ex, s.syncs); // K4
        bicg_update_p(p, rS, v, ex);                                         // K5
        return p4;
      }, decide);
      s.finish(param);
    }

    // ------------------------------------------------------------------ multi-shift CG (MdagM + sigma_j) with reliable updates
    // The CG-M recursion of the reference (lib/inv_multi_cg_quda.cpp): the Krylov space does not depend on the shift, so one
    // recursion on the smallest shift sigma_0 solves every shift for the operator cost of that one.  With CG's structure:
    // every scalar lives in one device block (blas::ms_scalars, run by the reduction finalisers), one iteration is
    // Ap = MdagM p_0, ms_dot, ms_update_r and ms_update_xp, and the host reads |r|^2, the active-shift count and the done
    // flag of iteration k - 1 while the GPU runs iteration k.  Shifts retire from the top; once all have, the kernels of the
    // iteration queued behind return at once, so the reported iteration count matches the solution.
    // Reliable updates (mixed precision) follow shift 0 with CG's criterion, as the reference's do: every x_j takes its
    // sloppy sum, r = b - (MdagM + sigma_0) x_0 is recomputed in the precise operator, and ms_replace_r repairs p_j with
    // zeta_j (r_true - r).  The residuals of the other shifts are then taken as zeta_j r_true; the drift that leaves is
    // what the single-shift refinement in invertMultiShiftCG removes.
    // More than one shift needs x_j = 0 on entry (collinear residuals); one shift may start from any x_0.
    static void multishift_cg(const Dirac &mat, const Dirac &matSloppy, std::vector<ColorSpinorField> &x, const ColorSpinorField &b,
                              MultiShiftParam &param)
    {
      using namespace blas;
      const int n = param.n_shift;
      Solve s(mat, matSloppy, &Dirac::MdagM, x[0], b);
      const Exec &ex = s.ex;
      s.shift = param.offset[0];
      Scratch Ap_s = s.sloppy();
      ColorSpinorField &Ap = Ap_s.f, &rS = s.rS;
      std::deque<Scratch> pool_p, pool_xS;
      std::vector<ColorSpinorField> p, xS, acc; // per shift: direction, sloppy solution, precise accumulator
      for (int j = 0; j < n; j++) {
        p.push_back(pool_p.emplace_back(ex.stream, x[0].X, s.sp, x[0].n_parity).f);
        xS.push_back(j == 0 ? s.xS : pool_xS.emplace_back(ex.stream, x[0].X, s.sp, x[0].n_parity).f);
        acc.push_back(j == 0 ? s.y : x[j]);
      }
      param.reliable_updates = 0;
      for (int j = 0; j < n; j++) {
        param.iter_offset[j] = param.refine_iter[j] = 0;
        param.iter_res_offset[j] = param.true_res_offset[j] = 0.0;
      }
      if (s.zero_source()) {
        param.iter = 0;
        s.complete(param);
        return;
      }

      double r2 = s.start();
      Scalars<M_COUNT> s0 {};
      s0.s[M_R2] = r2;
      for (int j = 0; j < n; j++) {
        if (j > 0) zero(xS[j], ex);
        copy(p[j], rS, ex);
        s0.s[M_DSIG + j] = param.offset[j] - param.offset[0];
        s0.s[M_ZETA + j] = s0.s[M_ZOLD + j] = s0.s[M_ALPHA + j] = 1.0;
        s0.s[M_STOP + j] = param.tol_offset[j] * param.tol_offset[j] * s.b2;
        s0.s[M_RES + j] = r2;
        s0.s[M_RETIRED + j] = -1.0;
      }
      int n_seen = n; // the active shifts as the host last saw them
      while (n_seen > 0 && r2 <= s0.s[M_STOP + n_seen - 1]) s0.s[M_RETIRED + --n_seen] = 0.0;
      s0.s[M_NACT] = n_seen;
      set_all<MsTraits>(ex, s0);
      const double stop = s0.s[M_STOP];
      CgReliable rel(r2);
      s.done = n_seen == 0;

      // convergence / reliable-update decision on the scalar block after iteration j; true if r was replaced
      auto decide = [&](const double *S, int j) {
        r2 = S[M_R2];
        n_seen = (int)S[M_NACT];
        const bool converged = S[M_DONE] != 0.0;
        if (converged) s.k = j; // the iteration queued after j returned at once
        if (!rel.update(r2, param.delta, !s.same_prec, converged)) {
          s.done = converged;
          return false;
        }
        // the shifts still active after iteration j take their sloppy sums now; a retired shift keeps its sum until the end
        for (int i = 1; i < n_seen; i++) {
          s.fold(acc[i], xS[i]);
          zero(xS[i], ex);
        }
        r2 = s.reliable_update();
        copy(Ap, s.r, ex); // the true residual in the sloppy precision; Ap is free until the next iteration
        ms_replace_r(p, rS, Ap, r2, ex);
        param.reliable_updates++;
        rel.reset(r2);
        s.done = r2 <= stop && n_seen <= 1;
        return true;
      };
      s.iterate<MsTraits>(param.maxiter, [&] {
        matSloppy.MdagM(Ap, p[0]);
        ms_dot(p[0], Ap, param.offset[0], ex, s.syncs);
        const Pending pr = ms_update_r(rS, Ap, ex, s.syncs);
        ms_update_xp(xS, p, rS, std::max(n_seen, 1), ex);
        return pr;
      }, decide);

      // every shift takes its sloppy sum; then the per-shift statistics and true residuals
      for (int j = 1; j < n; j++) s.fold(acc[j], xS[j]);
      s.fold();
      copy(x[0], s.y, ex);
      const std::vector<double> S = fetch<MsTraits>(ex);
      s.syncs++;
      for (int j = 0; j < n; j++) {
        s.shift = param.offset[j];
        param.true_res_offset[j] = std::sqrt(s.residual(x[j]) / s.b2);
        param.iter_res_offset[j] = std::sqrt(S[M_RES + j] / s.b2);
        param.iter_offset[j] = S[M_RETIRED + j] < 0.0 ? s.k : (int)S[M_RETIRED + j];
      }
      s.complete(param);
      param.iter = s.k;
    }

    void checkMultiShiftParam(const MultiShiftParam &param)
    {
      const int n = param.n_shift;
      if (n < 1 || n > B200_MAX_SHIFTS)
        throw Error("multi-shift CG: n_shift " + std::to_string(n) + " is outside 1.." + std::to_string(B200_MAX_SHIFTS));
      for (int j = 0; j < n; j++) {
        if (!std::isfinite(param.offset[j])) throw Error("multi-shift CG: offset " + std::to_string(j) + " is not finite");
        if (j > 0 && param.offset[j] < param.offset[j - 1])
          throw Error("multi-shift CG: the offsets must be non-decreasing (offset " + std::to_string(j) + " is below offset " +
                      std::to_string(j - 1) + ")");
        if (!(param.tol_offset[j] > 0.0)) throw Error("multi-shift CG: tol_offset " + std::to_string(j) + " must be > 0");
      }
    }

    // The public solve (invertMultiShiftQuda's order): the multi-shift recursion from x_j = 0, then every shift whose true
    // residual misses its tolerance is refined by the same solver with that single shift, starting from x_j -- which is CG
    // on MdagM + sigma_j with reliable updates.
    void invertMultiShiftCG(const Dirac &mat, const Dirac &matSloppy, std::vector<ColorSpinorField> &x, const ColorSpinorField &b,
                            MultiShiftParam &param)
    {
      checkMultiShiftParam(param);
      const int n = param.n_shift;
      if ((int)x.size() != n) throw Error("multi-shift CG: " + std::to_string(x.size()) + " solution fields for " + std::to_string(n) + " shifts");
      for (int j = 0; j < n; j++) {
        if (x[j].precision != mat.Precision()) throw Error("x and b must have the precise operator's precision");
        if (x[j].n_parity != b.n_parity || x[j].v == b.v) throw Error("multi-shift CG: each x_j must be a field of b's shape, apart from b");
        for (int i = 0; i < j; i++)
          if (x[i].v == x[j].v) throw Error("multi-shift CG: the solution fields must be distinct");
      }
      Solve::sloppy_precision(mat, matSloppy, x[0], b);
      for (ColorSpinorField &f : x) blas::zero(f, mat.exec());
      multishift_cg(mat, matSloppy, x, b, param);
      double secs = param.secs, flops = param.gflops * param.secs;
      for (int j = 0; j < n; j++) {
        if (!(param.true_res_offset[j] > param.tol_offset[j])) continue;
        MultiShiftParam one;
        one.n_shift = 1;
        one.offset[0] = param.offset[j];
        one.tol_offset[0] = param.tol_offset[j];
        one.maxiter = param.maxiter;
        one.delta = param.delta;
        std::vector<ColorSpinorField> xj {x[j]};
        multishift_cg(mat, matSloppy, xj, b, one);
        param.refine_iter[j] = one.iter;
        param.true_res_offset[j] = one.true_res_offset[0];
        param.reliable_updates += one.reliable_updates;
        param.host_syncs += one.host_syncs;
        secs += one.secs;
        flops += one.gflops * one.secs;
      }
      param.secs = secs;
      param.gflops = secs > 0.0 ? flops / secs : 0.0;
    }

  } // namespace host
} // namespace b200

