// TEST-ONLY host twin of the clover construction: twin_compute_clover / twin_clover_invert_packed forward to the same
// entry-point templates as libquda_b200's b200_compute_clover / b200_clover_invert_packed (quda_b200/csrc/clover_build.h:
// argument validation, site code) with a CPU executor that walks the kernels' grids (inst_clover_build.cu) site by site.
// It exists so that the CPU test tier checks the code the GPU runs; nothing under quda_b200/ loads it.
#include <cstdarg>
#include <cstdio>
#include <vector>

#include "../../quda_b200/csrc/clover_build.h"

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

  struct CloverTwin {
    static int require_device() { return 0; }

    // clover_build_kernel: one thread per site of each parity
    template <typename T> static int clover_build(const CloverBuildRequest &rq)
    {
      CloverBuildArgs<T> a;
      fill_clover_build(a, rq);
      for (int parity = 0; parity < 2; parity++)
#pragma omp parallel for
        for (int x_cb = 0; x_cb < a.volume_cb; x_cb++) clover_build_site(a, x_cb, parity);
      return 0;
    }

    // clover_invert_kernel + clover_trlog_kernel: per-CTA trees over kCloverBuildThreads sites, then one CTA per parity
    // that strides over the CTA partials and reduces them with the same tree
    template <typename T> static int clover_invert(const CloverInvertRequest &rq)
    {
      constexpr int B = kCloverBuildThreads;
      const int volume_cb = rq.X[0] * rq.X[1] * rq.X[2] * rq.X[3] / 2, nblk = (volume_cb + B - 1) / B;
      std::vector<double> partial(2 * (size_t)nblk);
      auto tree = [](double *s) {
        for (int w = B / 2; w > 0; w >>= 1)
          for (int tid = 0; tid < B; tid++) clover_tree_step(s, tid, w);
      };
      for (int parity = 0; parity < 2; parity++)
#pragma omp parallel for
        for (int b = 0; b < nblk; b++) {
          double s[B];
          for (int tid = 0; tid < B; tid++) {
            const int x_cb = b * B + tid;
            s[tid] = x_cb < volume_cb ? clover_invert_site((T *)rq.inv, (const T *)rq.packed, (size_t)parity * volume_cb + x_cb) : 0.0;
          }
          tree(s);
          partial[(size_t)parity * nblk + b] = s[0];
        }
      for (int parity = 0; parity < 2; parity++) {
        double s[B];
        for (int tid = 0; tid < B; tid++) {
          double v = 0.0;
          for (int i = tid; i < nblk; i += B) v += partial[(size_t)parity * nblk + i];
          s[tid] = v;
        }
        tree(s);
        rq.trlog[parity] = s[0];
      }
      return 0;
    }
  };
} // namespace b200

using namespace b200;

extern "C" {
const char *twin_last_error(void) { return g_err; }

int twin_compute_clover(void *packed, const void *const qdp[4], const int X[4], const int border[4], int precision, double coeff, void *stream)
{
  return compute_clover<CloverTwin>(packed, qdp, X, border, precision, coeff, stream);
}

int twin_clover_invert_packed(void *packed_inv, double trlog[2], const void *packed, const int X[4], int precision, void *stream)
{
  return clover_invert_packed<CloverTwin>(packed_inv, trlog, packed, X, precision, stream);
}
}
