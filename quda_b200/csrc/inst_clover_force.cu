// Kernels of b200_clover_force_accumulate (site code: clover_force.h).  Three launches on the caller's stream: the hopping
// force and the clover derivative each update mom once per (link, parity), one thread each; the sigma kernel writes the
// oprod field in between (one thread per site, parity and plane).  oprod is the only work field, stream-ordered scratch.
#include "clover_force.h"

namespace b200
{

  template <typename T> __global__ void __launch_bounds__(kCloverForceThreads) clover_hop_force_kernel(const CloverForceArgs<T> a)
  {
    const int x_cb = blockIdx.x * blockDim.x + threadIdx.x;
    if (x_cb >= a.volume_cb) return;
    clover_hop_force_site(a, x_cb, blockIdx.z, blockIdx.y);
  }

  template <typename T> __global__ void __launch_bounds__(kCloverForceThreads) clover_sigma_kernel(const CloverForceArgs<T> a)
  {
    const int x_cb = blockIdx.x * blockDim.x + threadIdx.x;
    if (x_cb >= a.volume_cb) return;
    clover_sigma_site(a, x_cb, blockIdx.y, blockIdx.z);
  }

  template <typename T> __global__ void __launch_bounds__(kCloverForceThreads) clover_deriv_kernel(const CloverForceArgs<T> a)
  {
    const int x_cb = blockIdx.x * blockDim.x + threadIdx.x;
    if (x_cb >= a.volume_cb) return;
    clover_deriv_site(a, x_cb, blockIdx.z, blockIdx.y);
  }

  template <typename T> int launch_clover_force(const CloverForceRequest &rq)
  {
    const int volume_cb = rq.X[0] * rq.X[1] * rq.X[2] * rq.X[3] / 2;
    cudaStream_t s = (cudaStream_t)rq.stream;
    T *oprod = nullptr; // [6][2 Vh][18]
    if (int rc = check_cuda(cudaMallocAsync((void **)&oprod, (size_t)6 * 2 * volume_cb * 18 * sizeof(T), s), "cudaMallocAsync")) return rc;
    CloverForceArgs<T> a;
    fill_clover_force(a, rq, oprod);
    const int nblk = (volume_cb + kCloverForceThreads - 1) / kCloverForceThreads;
    clover_hop_force_kernel<T><<<dim3(nblk, 4, 2), kCloverForceThreads, 0, s>>>(a);
    count_launch();
    clover_sigma_kernel<T><<<dim3(nblk, 2, 6), kCloverForceThreads, 0, s>>>(a);
    count_launch();
    clover_deriv_kernel<T><<<dim3(nblk, 4, 2), kCloverForceThreads, 0, s>>>(a);
    count_launch();
    int rc = check_cuda(cudaGetLastError(), "clover force launch");
    const int rf = check_cuda(cudaFreeAsync(oprod, s), "cudaFreeAsync");
    return rc ? rc : rf;
  }

  template int launch_clover_force<double>(const CloverForceRequest &);
  template int launch_clover_force<float>(const CloverForceRequest &);

} // namespace b200
