/*
 * b200_dslash.h -- C ABI of the H100 (sm_90a) Wilson / Wilson-clover Dslash engine (libquda_b200.so).
 *
 * This is the drop-in boundary for QUDA's Dslash free functions.  Each entry point names the reference
 * interface it replaces (paths relative to the lattice/quda tree); INTEGRATION.md shows the C++ shim that
 * fills these PODs from quda::ColorSpinorField / GaugeField / CloverField accessors.
 *
 * All pointers are DEVICE pointers unless stated otherwise.  Fields are in QUDA's native ("FloatN") orders
 * (include/color_spinor_field_order.h:1191-1300, include/gauge_field_order.h:1516-1588,
 * include/clover_field_order.h:587-720), spinors in the UKQCD gamma basis -- exactly what the reference
 * kernels consume, so resident QUDA fields can be passed unchanged.  Nothing is allocated per call; work is
 * enqueued on `stream` and the call returns without synchronising (as the reference does).
 *
 * Every function returns 0 on success or a negative b200_status; b200_last_error() gives the message
 * (the QUDA-side shim turns a non-zero status into errorQuda(), include/util_quda.h:73-78).
 */
#ifndef B200_DSLASH_H
#define B200_DSLASH_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_ABI_VERSION 3

typedef enum {
  B200_SUCCESS = 0,
  B200_ERR_INVALID = -1,     /* bad argument / unsupported combination */
  B200_ERR_CUDA = -2,        /* CUDA runtime error (launch, memcpy, IPC) */
  B200_ERR_UNSUPPORTED = -3, /* valid request outside the built instantiation set */
  B200_ERR_NO_DEVICE = -4    /* no usable CUDA device: the product has no CPU fallback */
} b200_status;

/* QudaPrecision values (include/enum_quda.h): bytes per real */
enum { B200_DOUBLE = 8, B200_SINGLE = 4, B200_HALF = 2 };

/* which operator; mirrors the three reference entry points */
typedef enum {
  B200_OP_WILSON = 0,   /* ApplyWilson:                    out = D in            | a != 0: out = x + a D in       */
  B200_OP_CLOVER = 1,   /* ApplyWilsonClover:              out = A x + a D in  (xpay form only)                   */
  B200_OP_CLOVER_PC = 2, /* ApplyWilsonCloverPreconditioned: out = A^-1 D in     | a != 0: out = x + a A^-1 D in  */
  /* degenerate twisted mass: the same stencil with a (1 + i b gamma5) rotation in the epilogue
   * (include/dslash_quda.h:363-406, include/kernels/dslash_twisted_mass*.cuh); b is negated for dagger */
  B200_OP_TWISTED_MASS = 3,   /* ApplyTwistedMass:  out = a D in + (1 + i b gamma5) x   (xpay form only, a != 0)       */
  B200_OP_TWISTED_MASS_PC = 4 /* ApplyTwistedMassPreconditioned: out = a (1 + i b gamma5) D in [+ x if x.v != NULL];
                               * dagger without `asymmetric`: out = D^dagger a (1 - i b gamma5) in [+ x]              */
} b200_op;

typedef enum {
  B200_KERNEL_AUTO = 0,     /* interior, then (if any comm_dim set) wait for halos and run the exterior update */
  B200_KERNEL_INTERIOR = 1, /* interior kernel only (hops across partitioned boundaries are skipped)           */
  B200_KERNEL_EXTERIOR = 2, /* fused exterior kernel only (adds ghost hops to the partial result in `out`)      */
  /* the two halves of B200_KERNEL_AUTO on a partitioned lattice, for callers that put them on different streams:  */
  B200_KERNEL_INTERIOR_TILES = 3, /* tiles that touch no partitioned face (independent of the halo)               */
  B200_KERNEL_BOUNDARY_TILES = 4, /* boundary tiles: waits for the arrival flags, then complete site updates      */
  /* the same split with 1-site-thick shells instead of whole boundary tiles (roles of the fused kernel without its pack role): */
  B200_KERNEL_INTERIOR_SITES = 5, /* every site that touches no partitioned face (independent of the halo)         */
  B200_KERNEL_BOUNDARY_SITES = 6  /* the face sites: waits for the arrival counters, then complete site updates    */
} b200_kernel;

/* One ColorSpinorField in native order.  n_parity == 1: a single-parity field (QUDA_PARITY_SITE_SUBSET);
 * n_parity == 2: full field, parity blocks `parity_stride_bytes` (= Bytes()/2) apart.
 * Half precision: `norm` may be NULL, in which case it is derived exactly like the reference accessor does,
 * (float*)((short*)v + 24*volume_cb), second parity parity_stride_bytes further on. */
typedef struct {
  void *v;
  void *norm;
  size_t parity_stride_bytes;
  int volume_cb;
  int n_parity;
} b200_spinor;

/* GaugeField in native order with the neighbour's backward links in the pad (QUDA_GHOST_EXCHANGE_PAD). */
typedef struct {
  const void *gauge;
  size_t parity_stride_bytes; /* Bytes()/2 */
  int stride;                 /* volume_cb + pad */
  int reconstruct;            /* 18, 12 or 8 */
  double anisotropy;          /* GaugeField::Anisotropy() */
  double link_max;            /* GaugeField::LinkMax(): fixed-point scale of reconstruct-18 half links */
  int t_boundary;             /* +1 periodic, -1 anti-periodic (QudaTboundary) */
  int first_time_slice;       /* comm_coord(3) == 0 */
  int last_time_slice;        /* comm_coord(3) == comm_dim(3)-1 */
} b200_gauge;

/* CloverField in native order (field holding A, or A^-1 when is_inverse). */
typedef struct {
  const void *clover;
  size_t parity_stride_bytes;
  int compressed;     /* clover::reconstruct(): 28 reals per chiral block instead of 36 */
  int dynamic_inverse; /* clover::dynamic_inverse(): field holds A; A^-1 is applied by per-site Cholesky solve */
  double diagonal;    /* CloverField::Diagonal() (compressed format only) */
  double max_element; /* CloverField::max_element(is_inverse) (fixed point only) */
} b200_clover;

/* Halo state for partitioned dimensions.  ghost[d][dir]: received, spin-projected faces for dimension d,
 * dir 0 = data that came from the backward neighbour (used by the x[d]==0 sites), dir 1 = from the forward
 * neighbour.  Layout per face: both parities back to back, each [M_ghost planes][face_cb] (+ float norms for
 * half precision) as in include/color_spinor_field_order.h:1065-1180. */
typedef struct {
  int comm_dim[4];
  void *ghost[4][2];
  void *ghost_norm[4][2]; /* half precision only; NULL -> directly after the 12*face_cb shorts of each parity block */
  /* Arrival flags (optional).  If wait_flag[d][dir] is non-NULL the boundary / exterior kernel spins until the 32-bit
   * site counter it points to (in THIS GPU's memory, advanced by the neighbour's pack CTAs over NVLink, see
   * b200_pack_args.signal) shows that exchange `seq` has landed: count >= ((seq + (seq & 1)) / 2) * face_cb[d], before it
   * reads ghost[d][dir].  NULL: arrival is guaranteed by stream order (copy-engine / NCCL path). */
  void *wait_flag[4][2];
  unsigned seq;
  int *timeout_flag; /* device word set to 1 if a wait gave up after ~10 s (never hangs the GPU); may be NULL */
  /* Multi-RHS batches (b200_dslash_apply_multi after b200_pack_ghost_multi): source i reads ghost[d][dir] (and ghost_norm)
   * + i * src_stride[d] bytes; wait_flag and seq are shared by the batch.  0 for single-source calls. */
  size_t src_stride[4];
} b200_halo;

typedef struct {
  int abi_version;    /* B200_ABI_VERSION */
  int op;             /* b200_op */
  int kernel;         /* b200_kernel */
  int precision;      /* B200_DOUBLE / B200_SINGLE / B200_HALF: storage precision of out/in/x/U/A */
  int X[4];           /* local lattice extents (full sites), all even */
  int parity;         /* destination parity (n_parity == 1); ignored for full fields */
  int dagger;
  double a;           /* 0 => no xpay (include/kernels/dslash_wilson.cuh:54); B200_OP_TWISTED_MASS_PC: scale of the rotation */
  double b;           /* twisted mass only: the twist factor (2 mu kappa, or -2 kappa mu for the inverse rotation) */
  int asymmetric;     /* B200_OP_TWISTED_MASS_PC only: asymmetric preconditioning (needs dagger, excludes x) */
  b200_spinor out, in, x;
  b200_gauge U;
  b200_clover A;      /* ignored for B200_OP_WILSON */
  b200_halo halo;
  int tile[4];        /* launch-geometry override (cb-sites in x, sites in y,z,t); all 0 => built-in default */
  void *stream;       /* cudaStream_t */
} b200_dslash_args;

/* replaces quda::ApplyWilson / ApplyWilsonClover / ApplyWilsonCloverPreconditioned
 * (include/dslash_quda.h:83,137,234; lib/dslash_wilson.cu:9-20) */
int b200_dslash_apply(const b200_dslash_args *args);

/* The multi-RHS form of the same three entry points: QUDA passes cvector_ref<ColorSpinorField> batches that share
 * one gauge (and clover) field (include/dslash_quda.h:83-234; WilsonArg::out/in/x[MAX_MULTI_RHS],
 * include/kernels/dslash_wilson.cuh:37-69; QUDA_MAX_MULTI_RHS defaults to 16, lib/CMakeLists.txt:298-300).
 * `args` is read as for b200_dslash_apply except that args->out / in / x are ignored in favour of out[i], in[i], x[i]
 * (x may be NULL when a == 0).  On an unpartitioned lattice each thread updates its site for up to 4 sources at once
 * (2 in fp64) with the links held in registers, so the link stream is read once per batch; with partitioned dimensions
 * or an explicit kernel selector the sources are applied one after the other, source i on its own ghost slab
 * (args->halo.src_stride, filled by ONE b200_pack_ghost_multi for the whole batch). */
#define B200_MAX_MULTI_RHS 16
int b200_dslash_apply_multi(const b200_dslash_args *args, int n_src, const b200_spinor *out, const b200_spinor *in,
                            const b200_spinor *x);

/* replaces quda::ApplyClover(out, in, clover, inverse, parity) (include/dslash_quda.h:811;
 * lib/dslash_clover_helper.cu:46-54): out = A in or A^-1 in on one parity */
int b200_clover_apply(const b200_spinor *out, const b200_spinor *in, const b200_clover *A, int precision, int inverse,
                      int parity, void *stream);

/* replaces quda::ApplyTwistGamma(out, in, 4, kappa, mu, 0, dagger, type) for the singlet flavour (include/dslash_quda.h:883,
 * include/kernels/dslash_gamma_helper.cuh:55-62): out = a (1 + i b gamma5) in on one parity, with
 * direct: b = 2 kappa mu, a = 1;  inverse: b = -2 kappa mu, a = 1 / (1 + b^2);  dagger negates b.  out may alias in. */
int b200_twist_gamma5(const b200_spinor *out, const b200_spinor *in, int precision, double kappa, double mu, int dagger,
                      int inverse, void *stream);

/* replaces quda::PackGhost (include/dslash_quda.h:919; lib/dslash_pack2.cu:55-425): spin-project the boundary
 * sites of `in` (parity 1-parity... see b200_pack_args) and store 12-real half spinors into the send targets,
 * which may be local buffers or peer-GPU ghost buffers mapped over NVLink. */
typedef struct {
  int abi_version;
  int precision;
  int X[4];
  int parity;      /* parity of the sites being packed (= the input parity of the Dslash that follows) */
  int dagger;
  b200_spinor in;
  int comm_dim[4];
  void *dst[4][2];      /* [d][0]: where our x[d]==0 face goes (the backward neighbour's ghost[d][1] slot);
                           [d][1]: where our x[d]==X[d]-1 face goes (the forward neighbour's ghost[d][0] slot) */
  void *dst_norm[4][2]; /* half precision */
  /* Remote-write completion signalling (QUDA_P2P_REMOTE_WRITE without MPI in the critical path, cf.
   * lib/dslash_policy.hpp:1682-1687, include/shmem_pack_helper.cuh:60-190): signal[d][f] is a 32-bit word in the
   * RECEIVER's memory that COUNTS the face sites that have landed in that ghost buffer since the exchange was set up
   * (per pack CTA: barrier, one system fence, a local ticket; the last CTA of the face stores the new total).  The buffer
   * pair is used alternately (buffer seq & 1), so exchange `seq` has arrived once the count reaches
   * ((seq + (seq & 1)) / 2) * face_cb.  `block_counter` is an 8-int zero-initialised scratch array in local device memory
   * (the tickets). */
  void *signal[4][2];
  int *block_counter;
  unsigned seq;
  void *stream;
} b200_pack_args;
int b200_pack_ghost(const b200_pack_args *args);

/* The batched (multi-RHS) form of PackGhost: the reference packs every source of a cvector_ref batch in ONE launch, the
 * source index riding in the thread grid (lib/dslash_pack2.cu:55-403; WilsonArg::in[MAX_MULTI_RHS],
 * include/kernels/dslash_wilson.cuh:37-40).  args->in is ignored in favour of in[0 .. n_src): source s is written
 * s * dst_stride[d] bytes behind args->dst[d][f] (and dst_norm), i.e. the receiver holds n_src ghost slabs per face,
 * dst_stride[d] >= one parity's face bytes apart.  args->signal[d][f] moves ONCE, to the same value as for the single
 * exchange `seq`, when the last site of the last source has landed; each source's Dslash then runs with
 * b200_halo.ghost[d][dir] + s * stride, the same wait_flag and the same seq.  One pack launch, one NVLink round trip and
 * one arrival signal per face for the whole batch. */
int b200_pack_ghost_multi(const b200_pack_args *args, int n_src, const b200_spinor *in, const size_t dst_stride[4]);

/* The whole partitioned Dslash -- what ApplyWilson* does on a partitioned lattice through its policy
 * (lib/dslash_wilson.hpp:18-54 -> lib/dslash_policy.hpp:1471-1650: pack, exchange, interior, exterior) -- as ONE kernel
 * launch on args->stream: pack CTAs write the faces of `in` into the neighbours' ghost slabs and raise their arrival
 * flags, interior CTAs update every site that touches no partitioned face meanwhile, boundary CTAs acquire the
 * neighbours' flags and update the face sites completely.  `pack` must describe the faces of args->in (parity
 * 1 - args->parity, same dagger / precision / lattice / partitioning, pack->seq == args->halo.seq); fields single parity.
 * args->kernel selects the roles of the launch: B200_KERNEL_AUTO all three; B200_KERNEL_INTERIOR_TILES the interior role
 * alone (independent of the halo) and B200_KERNEL_BOUNDARY_TILES pack + boundary, for callers that put the two halves on
 * different streams (the default schedule of this library's own operator layer: pack + boundary on a high-priority side
 * stream).  Without partitioned dimensions it is b200_dslash_apply(args). */
int b200_dslash_apply_fused(const b200_dslash_args *args, const b200_pack_args *pack);

/* bytes of one face buffer holding BOTH parities (what b200_halo.ghost[d][dir] must point to), and of one parity */
size_t b200_ghost_face_bytes(int precision, const int X[4], int dim);

/* Device-side spinor marshaling (the spinor slice of QUDA's copy kernels, lib/copy_color_spinor.cu,
 * include/kernels/copy_color_spinor.cuh:4-89): converts between the host interface order
 * (QUDA_SPACE_SPIN_COLOR_FIELD_ORDER: [site][spin 4][colour 3][re,im], DeGrand-Rossi basis, fp64 or fp32, one parity)
 * and the native FloatN order in the UKQCD basis at `native.` precision.  Both buffers are device memory.
 * to_native != 0: host order -> native;  to_native == 0: native -> host order. */
int b200_copy_spinor(const b200_spinor *native, int native_precision, void *host_order, int host_precision, int to_native,
                     void *stream);

/* Device-side gauge marshaling (the Wilson slice of lib/copy_gauge*.cu + lib/extract_gauge_ghost*.cu as used by
 * loadGaugeQuda, lib/interface_quda.cpp:571-764): host interface order QUDA_QDP_GAUGE_ORDER
 * (qdp[mu][(parity*volume_cb + x_cb)][3][3][2], fp64 or fp32, already resident on the device) -> native FloatN order
 * at `native_precision` with 18/12/8-parameter packing, and the pad of every direction filled with the backward
 * neighbour's boundary links.  ghost_links[mu] (may be NULL = this rank is its own neighbour in mu, i.e. periodic
 * wrap) points to those links in face order: [parity][face_cb][3][3][2] at host precision.
 * `native` must describe a buffer of 2 * parity_stride_bytes with stride = volume_cb + pad. */
int b200_copy_gauge(const b200_gauge *native, int native_precision, const int X[4], void *const qdp[4],
                    void *const ghost_links[4], int host_precision, void *stream);

/* Device-side clover marshaling (lib/copy_clover.cu): host packed order [site (parity-major)][2 chiral blocks][36]
 * (6 real diagonals + 15 complex strictly-lower entries, fp64 / fp32, on the device) -> native order holding A/2,
 * optionally compressed to 28 reals per block (native->compressed, native->diagonal) and, for half precision, scaled
 * by native->max_element. */
int b200_copy_clover(const b200_clover *native, int native_precision, const int X[4], const void *packed, int host_precision,
                     void *stream);

/* The clover term computed from the links (loadCloverQuda with compute_clover, lib/interface_quda.cpp:803-900):
 * packed[V][2][36] = A = 1 + coeff sum_{mu<nu} sigma_mu,nu F_mu,nu (clover-leaf F, both chiral blocks, packed order as
 * b200_copy_clover reads it), coeff = kappa * c_sw (QudaInvertParam::clover_coeff).  qdp[mu] are device QDP-order links
 * [2 Vh_e][3][3][2] of the extended lattice X_e = X + 2 border: border[d] = 0 wraps periodically inside the local block,
 * border[d] = 1 means the caller filled a depth-1 halo, corners included.  precision (8 or 4) is that of links and output. */
int b200_compute_clover(void *packed, const void *const qdp[4], const int X[4], const int border[4],
                        int precision /* 8 or 4: links and output */, double coeff, void *stream);
/* packed_inv = A^-1 by Cholesky in double (NULL: trlog only); trlog[p] = sum over parity-p sites and both chiralities of
 * log det A (a host array).  The sums are taken in a fixed order, so repeated calls give bit-identical values.
 * Synchronises the stream, as cloverInvert does for its reduction. */
int b200_clover_invert_packed(void *packed_inv, double trlog[2], const void *packed, const int X[4], int precision, void *stream);

/* Halo buffers that peer GPUs must be able to map: plain cudaMalloc allocations (zero-filled) plus CUDA-IPC
 * export / import.  Replaces the reference's static ghost buffers + IPC handle exchange
 * (lib/lattice_field.cpp:252-470, lib/targets/cuda/comm_target.cpp:37-167); the 64-byte handles travel between
 * ranks over whatever bootstrap the host uses (torch.distributed here, MPI in QUDA). */
#define B200_IPC_HANDLE_BYTES 64
int b200_comm_alloc(void **ptr, size_t bytes);
int b200_comm_free(void *ptr);
int b200_ipc_get_handle(void *ptr, unsigned char handle[B200_IPC_HANDLE_BYTES]);
int b200_ipc_open_handle(const unsigned char handle[B200_IPC_HANDLE_BYTES], void **peer_ptr);
int b200_ipc_close_handle(void *peer_ptr);
/* synchronous cudaMemcpy(dst, src, bytes, cudaMemcpyDefault) for the small control words living in comm memory */
int b200_comm_copy(void *dst, const void *src, size_t bytes);

/* ------------------------------------------------------------------------------------------------------------
 * Operator + solver layer ("next" rows of the scope table): the C++ classes in quda_b200/csrc/host/dirac.h mirror
 * DiracWilson[PC] / DiracClover[PC] (lib/dirac_wilson.cpp, lib/dirac_clover.cpp) and CG with reliable updates
 * (lib/inv_cg_quda.cpp); these entry points expose them to non-C++ hosts the way MatQuda / invertQuda
 * (include/quda.h:1206,1337) expose QUDA's. */
#define B200_MAX_RANKS 16
#define B200_REDUCE_SLOT_BYTES 64                                              /* 4 doubles + sequence word, padded */
#define B200_REDUCE_MAILBOX_BYTES (2 * B200_MAX_RANKS * B200_REDUCE_SLOT_BYTES) /* [buffer parity][source rank] */
typedef struct {
  int comm_dim[4];
  void *send_dst[2][4][2];    /* [buffer][dim][face] peer-mapped destination of our faces */
  void *send_signal[2][4][2]; /* matching arrival flags in the receivers' memory */
  void *recv[2][4][2];        /* [buffer][dim][dir] local ghost buffers */
  void *recv_flag[2][4][2];
  int *block_counter;
  int *timeout_flag;
  unsigned seq;               /* exchanges started so far (all ranks advance in lock step) */
  void *pack_stream;          /* optional cudaStream_t: pack kernels run there, concurrently with the interior tiles */
  void (*allreduce_sum)(double *data, int n, void *user); /* NULL on a single rank */
  void *user;
  /* Optional NVLink all-reduce for the solver's scalars (dot products / norms), replacing the host callback above and
   * the reference's MPI_Allreduce on the host (lib/reduce_quda.cu -> comm_allreduce_sum, lib/communicator_mpi.cpp):
   * reduce_peer[r] is rank r's mailbox region (B200_REDUCE_MAILBOX_BYTES, zero-initialised comm memory) as mapped into
   * THIS process, reduce_peer[rank] the local one.  Every rank remote-writes its partial sums into its slot of every
   * mailbox, raises the slot's sequence number (st.release.sys), waits for all slots of its own mailbox and adds them
   * in rank order -- so all ranks obtain bit-identical sums.  n_ranks == 0: not available, use allreduce_sum. */
  int rank, n_ranks;
  void *reduce_peer[B200_MAX_RANKS];
  unsigned reduce_seq; /* reductions done so far (all ranks advance in lock step) */
} b200_comm;

typedef struct b200_dirac_s b200_dirac; /* opaque */

typedef enum { B200_DIRAC_WILSON = 0, B200_DIRAC_WILSONPC = 1, B200_DIRAC_CLOVER = 2, B200_DIRAC_CLOVERPC = 3,
               B200_DIRAC_TWISTED_MASS = 4, B200_DIRAC_TWISTED_MASSPC = 5 /* singlet flavour, lib/dirac_twisted_mass.cpp */
} b200_dirac_type;
typedef enum { B200_MATPC_EVEN_EVEN = 0, B200_MATPC_ODD_ODD = 1, B200_MATPC_EVEN_EVEN_ASYMMETRIC = 2,
               B200_MATPC_ODD_ODD_ASYMMETRIC = 3 } b200_matpc_type;
typedef enum { B200_APPLY_M = 0, B200_APPLY_MDAG = 1, B200_APPLY_MDAGM = 2, B200_APPLY_DSLASH = 3,
               B200_APPLY_DSLASH_XPAY = 4 } b200_apply;

/* Dirac::create (lib/dirac.cpp).  `A`/`Ainv` may be NULL for Wilson; `comm` may be NULL on a single rank.  The
 * descriptors are copied; the fields they point to stay owned by the caller and must outlive the operator. */
int b200_dirac_create(b200_dirac **op, int type, int precision, const int X[4], const b200_gauge *U, const b200_clover *A,
                      const b200_clover *Ainv, double kappa, int matpc_type, b200_comm *comm, void *stream);
/* twisted-mass operators: the twist mass mu (DiracParam::mu); 0 after creation */
int b200_dirac_set_twist(b200_dirac *op, double mu);
int b200_dirac_destroy(b200_dirac *op);
/* M / Mdag / MdagM act on full fields (unpreconditioned types) or single-parity fields (PC types);
 * DSLASH / DSLASH_XPAY take the destination parity, x and k as Dirac::Dslash[Xpay] do. */
int b200_dirac_apply(b200_dirac *op, int what, const b200_spinor *out, const b200_spinor *in, int parity,
                     const b200_spinor *x, double k, int dagger);
/* Halo health check: B200_SUCCESS if no halo wait has given up since the last check on this exchange, an error (flag
 * cleared) otherwise; synchronises `stream`.  Kernels waiting for a neighbour's faces give up after ~10 s of SM clocks so
 * that a lost peer can never hang the GPU; b200_invert_cg checks by itself, other callers check at their sync points. */
int b200_comm_check(b200_comm *comm, void *stream);
/* Dirac::prepare / Dirac::reconstruct for a full-system solve through the preconditioned operator: src_parity /
 * sol_parity receive which parity block of x holds the preconditioned source / solution. */
int b200_dirac_prepare(b200_dirac *op, const b200_spinor *x, const b200_spinor *b, int *src_parity, int *sol_parity);
int b200_dirac_reconstruct(b200_dirac *op, const b200_spinor *x, const b200_spinor *b);

typedef struct {
  double tol;       /* relative residual target |r|/|b| */
  int maxiter;
  double delta;     /* reliable-update threshold */
  int iter;         /* out */
  int reliable_updates;
  double true_res;  /* out: |b - A x| / |b| recomputed in the precise operator */
  double secs, gflops;
  int host_syncs;   /* out: stream synchronisations during the solve (~1 per iteration, one iteration behind the GPU) */
} b200_solver_param;
/* CG on MdagM x = b (x, b in the precise operator's precision; sloppy may equal precise) */
int b200_invert_cg(b200_dirac *precise, b200_dirac *sloppy, const b200_spinor *x, const b200_spinor *b, b200_solver_param *param);
/* BiCGStab on M x = b with the operator as given (the preconditioned system for the *pc types, the full one otherwise);
 * same fields and precisions as b200_invert_cg, restarts after a breakdown are counted in reliable_updates */
int b200_invert_bicgstab(b200_dirac *precise, b200_dirac *sloppy, const b200_spinor *x, const b200_spinor *b, b200_solver_param *param);

#define B200_MAX_SHIFTS 32 /* shifts of one multi-shift solve (QUDA_MAX_MULTI_SHIFT) */
typedef struct {
  int n_shift;                              /* 1 .. B200_MAX_SHIFTS */
  double offset[B200_MAX_SHIFTS];           /* sigma_j: finite, non-decreasing */
  double tol_offset[B200_MAX_SHIFTS];       /* per-shift relative residual target, > 0 */
  int maxiter;                              /* of the multi-shift loop and of each refinement solve */
  double delta;                             /* reliable-update threshold */
  int iter;                                 /* out: multi-shift iterations */
  int iter_offset[B200_MAX_SHIFTS];         /* out: iteration at which shift j retired */
  int refine_iter[B200_MAX_SHIFTS];         /* out: iterations of shift j's single-shift refinement (0: none needed) */
  double iter_res_offset[B200_MAX_SHIFTS];  /* out: iterated residual zeta_j |r| / |b| when shift j retired */
  double true_res_offset[B200_MAX_SHIFTS];  /* out: |b - (A + sigma_j) x_j| / |b| in the precise operator */
  int reliable_updates;
  double secs, gflops;
  int host_syncs;
} b200_multishift_param;
/* Multi-shift CG: (MdagM + sigma_j) x_j = b for every shift at once (the preconditioned system for the *pc types, the full one
 * otherwise).  x points to n_shift descriptors; every x_j is overwritten (the initial guess is ignored).  Shifts whose true
 * residual misses tol_offset[j] are refined by a single-shift solve from x_j. */
int b200_invert_multishift_cg(b200_dirac *precise, b200_dirac *sloppy, const b200_spinor *x, const b200_spinor *b,
                              b200_multishift_param *param);

/* The clover fermion force (computeCloverForceQuda -> computeCloverForce, lib/interface_quda.cpp:4539-4612,
 * lib/clover_force.cpp): non-twisted Wilson-clover, asymmetric even-odd preconditioning, MATPCDAG_MATPC solutions, no
 * determinant ratio, one GPU (no partitioned dimension).
 *
 * Kernel level.  mom[V][4][10] (parity-major sites; per link the (01), (02), (12) complex entries, the three imaginary
 * diagonals and one pad real, the reference's QUDA_ASQTAD_MOM_LINKS order) is updated in place:
 *   mom -= TA( U_mu(x) sum_i force_coeff[i] tr_spin[(1+g_mu) x_i(x+mu) p_i(x)^+ + (1-g_mu) p_i(x+mu) x_i(x)^+]
 *            + clover derivative of oprod ),
 *   oprod_mu,nu = sum_i epsilon[i][parity] (R_i - R_i^+), R_i = tr_spin[sigma_nu,mu x_i p_i^+],
 *                 plus sigma_coeff tr_spin[sigma_mu,nu A^-1] on the sites of parity trlog_parity,
 * TA = traceless anti-Hermitian part.  x[i], p[i] are full-lattice (both parities) native spinors, 1 <= n <=
 * B200_MAX_SHIFTS; qdp[mu] are the device QDP-order links [V][3][3][2] (boundary signs included, as b200_compute_clover
 * takes them); packed is A [V][2][36] as b200_compute_clover writes it.  Everything is in `precision` (8 or 4).
 * Asynchronous on `stream`. */
int b200_clover_force_accumulate(void *mom, const void *const qdp[4], const void *packed, const int X[4], int precision, int n,
                                 const void *const *x, const void *const *p, const double *force_coeff,
                                 const double *epsilon /* [n][2] */, double sigma_coeff, int trlog_parity, void *stream);
/* Operator level, the arguments of computeCloverForceQuda: mom as above, x[i] the n single-parity solutions (of the
 * operator's parity) of (Mhat^+ Mhat + sigma_i) x_i = phi as b200_invert_multishift_cg writes them, coeff[i] their residues,
 * kappa2 = -kappa^2 and ck = -c_sw kappa / 8 as MILC passes them, qdp and packed as above.  op must be a "cloverpc"
 * operator with asymmetric matpc on an unpartitioned lattice (B200_ERR_INVALID otherwise).  It prepares p_i and the other
 * parity of x_i on the operator's stream in scratch fields, along the reference's dagger branch (for these solutions the
 * non-dagger branch is the force of the Mhat Mhat^+ action), then adds the force with force_coeff = 2 dt coeff kappa2,
 * epsilon = 2 ck coeff dt on the operator's parity and -kappa2 2 ck coeff dt on the other, and sigma_coeff =
 * 2 ck multiplicity dt on the other parity: the update is the derivative of
 * sum_i coeff_i phi^+ (Mhat^+ Mhat + sigma_i)^-1 phi - multiplicity tr log A_other.  Synchronises the operator's stream. */
int b200_clover_force(void *mom, double dt, const b200_spinor *x, const double *coeff, double kappa2, double ck, int n,
                      double multiplicity, const void *const qdp[4], const void *packed, b200_dirac *op);

/* The gauge half of an HMC step on one GPU (no partitioned dimension): computeGaugeForceQuda, updateGaugeFieldQuda,
 * momActionQuda and plaqQuda (lib/interface_quda.cpp).  Fields as for the clover force: qdp[mu] are device QDP-order links
 * [V][3][3][2] with the fermion boundary sign included (every closed loop crosses the t boundary an even number of times,
 * so the sign cancels in the force and the plaquette, and exp(dt P)(-U) = -exp(dt P) U keeps it through the update); mom is
 * [V][4][10] as above.  Sites are parity-major, neighbours wrap periodically.  precision is 8 or 4 for every field.
 *
 * Gauge force: for every link U_mu(x),
 *   mom <- TA(mom - eb3 U_mu(x) sum_i coeff[i] path_i),
 * path_i the ordered product of the links of paths[mu][i][0 .. length[i]) (steps 0..3 forward along that direction, 7 - d
 * backward along d) walked from x + mu-hat; it must end at x.  paths is a flat int array [4][num_paths][max_length];
 * length and coeff have num_paths entries.  The path table travels in the kernel's parameter block, which bounds it:
 * 1 <= num_paths <= B200_GAUGE_MAX_PATHS, 1 <= length[i] <= max_length <= B200_GAUGE_MAX_LENGTH.  Steps outside 0..7
 * and open paths are refused.  Asynchronous on `stream`. */
#define B200_GAUGE_MAX_PATHS 64  /* the Symanzik set (plaquette, rectangle and parallelogram staples) has 48 */
#define B200_GAUGE_MAX_LENGTH 12 /* steps per path after the first link U_mu(x) */
int b200_gauge_force(void *mom, const void *const qdp[4], const int X[4], int precision, const int *paths, const int *length,
                     const double *coeff, int num_paths, int max_length, double eb3, void *stream);
/* out[mu] = exp(dt P) in[mu] for every link, P the traceless part of mom (conj_mom: of its adjoint).  exact = 1: the closed
 * form of the SU(3) exponential (Cayley-Hamilton, Morningstar & Peardon hep-lat/0311018); exact = 0: the order-8 Taylor
 * expansion of the reference (Horner form).  out may be in.  Asynchronous on `stream`. */
int b200_update_gauge(void *const out[4], const void *const in[4], const void *mom, const int X[4], int precision, double dt,
                      int conj_mom, int exact, void *stream);
/* *S = sum over links of 1/2 sum_k (Im P_kk)^2 + sum_{i<j} |P_ij|^2 - 4 (MILC's normalisation), summed in double in a
 * fixed order: repeated calls give identical sums.  Synchronises `stream`. */
int b200_mom_action(double *S, const void *mom, const int X[4], int precision, void *stream);
/* plaq = {total, spatial, temporal}: the mean of Re tr P_mu,nu / 3 over the sites and the three spatial (mu, nu < 3),
 * resp. temporal planes; total = (spatial + temporal) / 2.  Fixed-order double sums; synchronises `stream`. */
int b200_plaquette(double plaq[3], const void *const qdp[4], const int X[4], int precision, void *stream);

/* The gradient flow of a gauge field (performWFlowQuda) and its clover observables (gaugeObservablesQuda), on one GPU with
 * the fields of the gauge force above.
 *
 * Gradient flow: n_steps steps of Lüscher's RK3 integrator (arXiv:1006.4518, App. C) at step size epsilon (negative:
 * the flow backwards) of dV/dt = Z(V) V with the generator Z_mu(x) = -TA(U_mu(x) sum_i coeff[i] path_i), the path table
 * as for b200_gauge_force, so the flow follows the action sum_i coeff[i] sum_loops Re tr(1 - loop_i).  The plaquette
 * staples with coeff 1 give the Wilson flow; plaquette 5/3 and rectangle -1/12 the Symanzik (Lüscher-Weisz) flow.  Every
 * closed loop crosses the t boundary an even number of times and exp(Z)(-U) = -exp(Z) U, so the links keep the fermion
 * boundary sign.  out may be in; in is otherwise left unchanged.  Scratch (one link field and [V][4][10]) is allocated
 * and freed stream-ordered.  Asynchronous on `stream`. */
int b200_gauge_flow(void *const out[4], const void *const in[4], const int X[4], int precision, const int *paths,
                    const int *length, const double *coeff, int num_paths, int max_length, double epsilon, int n_steps,
                    void *stream);
/* From the clover F_mu,nu = (Q - Q^+) / 8 of the six planes (10, 20, 21, 30, 31, 32): energy = {total, spatial, temporal},
 * spatial and temporal the sums over the sites and the planes with mu < 3, resp. mu = 3, of -Re tr(F^2) (F without its
 * trace) over V; *qcharge = sum_x q(x), q(x) = -1/(4 pi^2) Re (tr F10 F32 - tr F20 F31 + tr F21 F30), written to the
 * device array density[V] (parity-major; NULL: not written).  Fixed-order double sums; synchronises `stream`. */
int b200_gauge_observables(double energy[3], double *qcharge, double *density, const void *const qdp[4], const int X[4],
                           int precision, void *stream);

/* Gauge smearing (performGaugeSmearQuda's four kinds), on one GPU with the fields of the gauge force above.  S_mu(x) is the
 * sum of the staples of U_mu(x) over the smeared planes; d = 4, or 3 with 0 <= dir_ignore <= 3, which smears only the
 * other three directions (their staples leave the ignored direction out) and copies the ignored direction's links bit for
 * bit.  dir_ignore = -1 or 4: all four directions.  P[W] is the SU(3) projection: the unitary polar factor of W by Newton's
 * iteration (to 2e-15 in fp64, 1e-6 in fp32, at most 100 iterations) over the principal cube root of its determinant.
 *   B200_SMEAR_APE           coeff {alpha}:    U' = P[(1 - alpha) 1 + alpha / (2 (d - 1)) S U^+] U
 *   B200_SMEAR_STOUT         coeff {rho}:      U' = exp(rho TA(S U^+)) U
 *   B200_SMEAR_OVRIMP_STOUT  coeff {rho, eps}: the same with (5 - 2 eps) / 3 S - (1 - eps) / 12 R, R the 2x1 rectangle
 *                                              staples (Moran & Leinweber, arXiv:0801.1165)
 *   B200_SMEAR_HYP           coeff {alpha1, alpha2, alpha3}: Hasenfratz & Knechtli (hep-lat/0103029), every level
 *                            P[(1 - alpha) 1 + c staples U^+] U; 4-d: alpha3 / 2, alpha2 / 4, alpha1 / 6; 3-d: alpha3 / 2,
 *                            alpha2 / 4 (alpha1 unused)
 * The projection of the product with U^+ and exp(X)(-U) = -exp(X) U keep the fermion boundary sign.  n_steps >= 1 steps;
 * out may be in, which is otherwise unchanged.  Scratch is allocated and freed stream-ordered: the d smeared directions of
 * one link field unless the call is one step out of place, plus for HYP the decorated links, 2 x 12 links per site in 4-d
 * (3.6 GB at 32^4 in fp64) and 6 in 3-d.  Asynchronous on `stream`. */
#define B200_SMEAR_APE 0
#define B200_SMEAR_STOUT 1
#define B200_SMEAR_OVRIMP_STOUT 2
#define B200_SMEAR_HYP 3
int b200_gauge_smear(void *const out[4], const void *const in[4], const int X[4], int precision, int type, const double coeff[3],
                     int dir_ignore, int n_steps, void *stream);

const char *b200_last_error(void);
int b200_abi_version(void);
/* number of kernels this library has launched since load (bench.py's gpu_launches evidence) */
long b200_launch_count(void);
void b200_reset_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif
