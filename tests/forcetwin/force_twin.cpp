// TEST-ONLY host twin of the clover force: twin_clover_force_accumulate forwards to the same entry-point template as
// libquda_b200's b200_clover_force_accumulate (quda_b200/csrc/clover_force.h: argument validation, site code) with a CPU
// executor that walks the grids of the three kernels of inst_clover_force.cu site by site.  It exists so that the CPU test
// tier checks the code the GPU runs; nothing under quda_b200/ loads it.
#include <cstdarg>
#include <cstdio>
#include <vector>

#include "../../quda_b200/csrc/clover_force.h"

namespace b200
{
  static char g_err[512] = "";
  int set_error(int code, const char *fmt, ...)
  {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
  }
  int check_cuda(cudaError_t, const char *) { return 0; }
  void count_launch() { }

  struct ForceTwin {
    static int require_device() { return 0; }

    // clover_hop_force_kernel, clover_sigma_kernel, clover_deriv_kernel in launch order; oprod is the kernels' scratch
    template <typename T> static int clover_force(const CloverForceRequest &rq)
    {
      const int volume_cb = rq.X[0] * rq.X[1] * rq.X[2] * rq.X[3] / 2;
      std::vector<T> oprod((size_t)6 * 2 * volume_cb * 18);
      CloverForceArgs<T> a;
      fill_clover_force(a, rq, oprod.data());
      for (int parity = 0; parity < 2; parity++)
        for (int mu = 0; mu < 4; mu++)
#pragma omp parallel for
          for (int x_cb = 0; x_cb < volume_cb; x_cb++) clover_hop_force_site(a, x_cb, parity, mu);
      for (int p = 0; p < 6; p++)
        for (int parity = 0; parity < 2; parity++)
#pragma omp parallel for
          for (int x_cb = 0; x_cb < volume_cb; x_cb++) clover_sigma_site(a, x_cb, parity, p);
      for (int parity = 0; parity < 2; parity++)
        for (int mu = 0; mu < 4; mu++)
#pragma omp parallel for
          for (int x_cb = 0; x_cb < volume_cb; x_cb++) clover_deriv_site(a, x_cb, parity, mu);
      return 0;
    }
  };
} // namespace b200

using namespace b200;

extern "C" {
const char *twin_last_error(void) { return g_err; }

int twin_clover_force_accumulate(void *mom, const void *const qdp[4], const void *packed, const int X[4], int precision, int n,
                                 const void *const *x, const void *const *p, const double *force_coeff, const double *epsilon,
                                 double sigma_coeff, int trlog_parity, void *stream)
{
  return clover_force_accumulate<ForceTwin>(mom, qdp, packed, X, precision, n, x, p, force_coeff, epsilon, sigma_coeff,
                                            trlog_parity, stream);
}
}
