// C ABI of libquda_b200.so (declared in include/b200_dslash.h).  Plain pointers and sizes only.  The Dslash, pack,
// clover and twist entry points forward to plan.h's templates, with the CUDA launchers as their executor.
#include <atomic>
#include <cstdlib>
#include <cstring>

#include "plan.h"

namespace b200
{
  static thread_local char g_err[512] = "";
  static std::atomic<long> g_launches {0};

  int set_error(int code, const char *fmt, ...)
  {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
  }

  int check_cuda(cudaError_t e, const char *what)
  {
    if (e == cudaSuccess) return B200_SUCCESS;
    return set_error(B200_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
  }

  void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

  int require_device()
  {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
      cudaGetLastError();
      return set_error(B200_ERR_NO_DEVICE, "no CUDA device available: libquda_b200 has no CPU path (%s)",
                       e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    }
    return 0;
  }

  // the executor of plan.h's entry points: the per-precision CUDA launchers (inst_*.cu)
  struct Cuda {
    static int require_device() { return b200::require_device(); }
    template <class P> static int dslash(const LaunchRequest &rq) { return launch_precision<P>(rq); }
    template <class P> static int tma(const LaunchRequest &rq) { return launch_tma_precision<P>(rq); }
    template <class P> static int mrhs(const MrhsRequest &rq) { return launch_mrhs_precision<P>(rq); }
    template <class P> static int clover(const CloverRequest &rq) { return launch_clover_precision<P>(rq); }
    template <class P> static int twist(const TwistRequest &rq) { return launch_twist_precision<P>(rq); }
    template <class P> static int pack(const PackRequest &rq) { return launch_pack_precision<P>(rq); }
    template <class P> static int pack_multi(const PackRequest &rq, const PackBatchRequest &b) { return launch_pack_multi_precision<P>(rq, b); }
  };

} // namespace b200

using namespace b200;

extern "C" {

const char *b200_last_error(void) { return g_err; }
int b200_abi_version(void) { return B200_ABI_VERSION; }
long b200_launch_count(void) { return g_launches.load(); }
void b200_reset_launch_count(void) { g_launches.store(0); }

size_t b200_ghost_face_bytes(int precision, const int X[4], int dim)
{
  return 2 * ghost_parity_bytes(precision, X, dim);
}

int b200_dslash_apply(const b200_dslash_args *a) { return apply_dslash<Cuda>(a); }

int b200_dslash_apply_multi(const b200_dslash_args *a, int n_src, const b200_spinor *out, const b200_spinor *in,
                            const b200_spinor *x)
{
  return apply_dslash_multi<Cuda>(a, n_src, out, in, x);
}

int b200_clover_apply(const b200_spinor *out, const b200_spinor *in, const b200_clover *A, int precision, int inverse,
                      int parity, void *stream)
{
  return clover_apply<Cuda>(out, in, A, precision, inverse, parity, stream);
}

int b200_twist_gamma5(const b200_spinor *out, const b200_spinor *in, int precision, double kappa, double mu, int dagger,
                      int inverse, void *stream)
{
  return twist_gamma5<Cuda>(out, in, precision, kappa, mu, dagger, inverse, stream);
}

int b200_copy_spinor(const b200_spinor *native, int native_precision, void *host_order, int host_precision, int to_native,
                     void *stream)
{
  if (!native || !native->v || !host_order) return set_error(B200_ERR_INVALID, "b200_copy_spinor: null argument");
  if (int rc = require_device()) return rc;
  if (native->n_parity != 1) return set_error(B200_ERR_INVALID, "b200_copy_spinor converts one parity block per call");
  if (host_precision != B200_DOUBLE && host_precision != B200_SINGLE)
    return set_error(B200_ERR_INVALID, "host order precision must be 8 or 4 (got %d)", host_precision);
  CopyRequest rq;
  rq.native = native->v;
  rq.native_norm = native->norm;
  rq.host = host_order;
  rq.volume_cb = native->volume_cb;
  rq.host_precision = host_precision;
  rq.to_native = to_native ? 1 : 0;
  rq.stream = stream;
  switch (native_precision) {
  case B200_DOUBLE: return launch_copy_precision<PrecF64>(rq);
  case B200_SINGLE: return launch_copy_precision<PrecF32>(rq);
  case B200_HALF: return launch_copy_precision<PrecH16>(rq);
  }
  return set_error(B200_ERR_INVALID, "precision %d not in {8,4,2}", native_precision);
}

int b200_copy_gauge(const b200_gauge *native, int native_precision, const int X[4], void *const qdp[4],
                    void *const ghost_links[4], int host_precision, void *stream)
{
  if (!native || !native->gauge || !X || !qdp) return set_error(B200_ERR_INVALID, "b200_copy_gauge: null argument");
  if (int rc = require_device()) return rc;
  if (host_precision != B200_DOUBLE && host_precision != B200_SINGLE)
    return set_error(B200_ERR_INVALID, "host gauge precision must be 8 or 4 (got %d)", host_precision);
  GaugeCopyRequest rq;
  rq.native = *native;
  for (int d = 0; d < 4; d++) {
    if (X[d] < 2 || (X[d] & 1)) return set_error(B200_ERR_INVALID, "X[%d]=%d must be even and >= 2", d, X[d]);
    rq.X[d] = X[d];
    if (!qdp[d]) return set_error(B200_ERR_INVALID, "qdp[%d] is NULL", d);
    rq.qdp[d] = qdp[d];
    rq.ghost[d] = ghost_links ? ghost_links[d] : nullptr;
  }
  if (native_precision == B200_HALF && native->reconstruct == 18 && !(native->link_max > 0.0))
    return set_error(B200_ERR_INVALID, "half recon-18 needs link_max > 0");
  rq.host_precision = host_precision;
  rq.stream = stream;
  switch (native_precision) {
  case B200_DOUBLE: return launch_gauge_copy_precision<PrecF64>(rq);
  case B200_SINGLE: return launch_gauge_copy_precision<PrecF32>(rq);
  case B200_HALF: return launch_gauge_copy_precision<PrecH16>(rq);
  }
  return set_error(B200_ERR_INVALID, "precision %d not in {8,4,2}", native_precision);
}

int b200_copy_clover(const b200_clover *native, int native_precision, const int X[4], const void *packed, int host_precision,
                     void *stream)
{
  if (!native || !native->clover || !X || !packed) return set_error(B200_ERR_INVALID, "b200_copy_clover: null argument");
  if (int rc = require_device()) return rc;
  if (host_precision != B200_DOUBLE && host_precision != B200_SINGLE)
    return set_error(B200_ERR_INVALID, "host clover precision must be 8 or 4 (got %d)", host_precision);
  if (native_precision == B200_HALF && !(native->max_element > 0.0))
    return set_error(B200_ERR_INVALID, "half precision clover needs max_element > 0");
  CloverCopyRequest rq;
  rq.native = *native;
  for (int d = 0; d < 4; d++) rq.X[d] = X[d];
  rq.packed = packed;
  rq.host_precision = host_precision;
  rq.stream = stream;
  switch (native_precision) {
  case B200_DOUBLE: return launch_clover_copy_precision<PrecF64>(rq);
  case B200_SINGLE: return launch_clover_copy_precision<PrecF32>(rq);
  case B200_HALF: return launch_clover_copy_precision<PrecH16>(rq);
  }
  return set_error(B200_ERR_INVALID, "precision %d not in {8,4,2}", native_precision);
}

int b200_comm_alloc(void **ptr, size_t bytes)
{
  if (!ptr || bytes == 0) return set_error(B200_ERR_INVALID, "b200_comm_alloc: null pointer or zero size");
  if (int rc = require_device()) return rc;
  if (int rc = check_cuda(cudaMalloc(ptr, bytes), "cudaMalloc")) return rc;
  return check_cuda(cudaMemset(*ptr, 0, bytes), "cudaMemset");
}

int b200_comm_free(void *ptr) { return check_cuda(cudaFree(ptr), "cudaFree"); }

int b200_ipc_get_handle(void *ptr, unsigned char handle[B200_IPC_HANDLE_BYTES])
{
  static_assert(sizeof(cudaIpcMemHandle_t) == B200_IPC_HANDLE_BYTES, "IPC handle size");
  cudaIpcMemHandle_t h;
  if (int rc = check_cuda(cudaIpcGetMemHandle(&h, ptr), "cudaIpcGetMemHandle")) return rc;
  memcpy(handle, &h, sizeof(h));
  return B200_SUCCESS;
}

int b200_ipc_open_handle(const unsigned char handle[B200_IPC_HANDLE_BYTES], void **peer_ptr)
{
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, sizeof(h));
  return check_cuda(cudaIpcOpenMemHandle(peer_ptr, h, cudaIpcMemLazyEnablePeerAccess), "cudaIpcOpenMemHandle");
}

int b200_ipc_close_handle(void *peer_ptr) { return check_cuda(cudaIpcCloseMemHandle(peer_ptr), "cudaIpcCloseMemHandle"); }

int b200_comm_copy(void *dst, const void *src, size_t bytes)
{
  return check_cuda(cudaMemcpy(dst, src, bytes, cudaMemcpyDefault), "cudaMemcpy");
}

int b200_pack_ghost(const b200_pack_args *a) { return pack_ghost<Cuda>(a); }

int b200_pack_ghost_multi(const b200_pack_args *a, int n_src, const b200_spinor *in, const size_t dst_stride[4])
{
  return pack_ghost_multi<Cuda>(a, n_src, in, dst_stride);
}

int b200_dslash_apply_fused(const b200_dslash_args *a, const b200_pack_args *p) { return apply_dslash_fused<Cuda>(a, p); }
}
