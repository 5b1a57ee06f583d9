// TEST-ONLY host twin of the gradient flow and the gauge observables: twin_gauge_flow / twin_gauge_observables forward to
// the same entry-point templates as libquda_b200's b200_gauge_flow / b200_gauge_observables (quda_b200/csrc/gauge_flow.h:
// argument validation, site code, stage plan) with a CPU executor that walks the grids of the kernels of
// inst_gauge_flow.cu site by site and sums in the kernels' order.  It is built on the gauge twin (tests/gaugetwin), whose
// executor and entry points it includes, so one library serves the flow and the gauge force, momentum action and plaquette
// the flow tests use.  Nothing under quda_b200/ loads it.
#include <cstring>
#include <limits>

#include "../../quda_b200/csrc/gauge_flow.h"
#include "../gaugetwin/gauge_twin.cpp"

namespace b200
{
  struct FlowTwin : GaugeTwin {
    // gauge_flow_kernel, one grid (blocks, mu, parity) per RK3 stage, ping-ponging as launch_gauge_flow does; every thread
    // writes only its own link of the stage's output and its own accumulator entry
    template <typename T> static int gauge_flow(const GaugeFlowRequest &rq)
    {
      const size_t V = (size_t)rq.X[0] * rq.X[1] * rq.X[2] * rq.X[3];
      std::vector<T> scratch((4 * 18 + 4 * 10) * V, std::numeric_limits<T>::quiet_NaN()); // as uninitialised device memory
      void *tmp[4];
      for (int d = 0; d < 4; d++) tmp[d] = scratch.data() + d * V * 18;
      void *acc = scratch.data() + 4 * V * 18;
      const FlowPlan plan = flow_plan(rq);
      const void *src[4];
      for (int d = 0; d < 4; d++) src[d] = rq.in[d];
      for (int s = 0; s < plan.stages; s++) {
        void *const *dst = plan.writes_scratch(s) ? tmp : rq.out;
        GaugeFlowArgs<T> a;
        fill_flow_stage(a, rq, s, src, dst, acc);
        for (int parity = 0; parity < 2; parity++)
          for (int mu = 0; mu < 4; mu++)
#pragma omp parallel for
            for (int x_cb = 0; x_cb < a.f.g.volume_cb; x_cb++) gauge_flow_site(a, x_cb, parity, mu);
        for (int d = 0; d < 4; d++) src[d] = dst[d];
      }
      if (plan.ends_in_scratch())
        for (int d = 0; d < 4; d++) std::memcpy(rq.out[d], tmp[d], V * 18 * sizeof(T));
      return 0;
    }

    // gauge_obs_kernel's groups g[kind][parity]: every kind is reduced by its own per-CTA tree and second stage, so the
    // energies (kinds 0, 1) and the charge (kind 2) can go through the gauge twin's two-stage sum separately
    template <typename T> static int gauge_observables(const GaugeObsRequest &rq, double g[6])
    {
      CloverBuildArgs<T> a;
      fill_lattice(a, rq.qdp, rq.X);
      two_stage(a.volume_cb, 2, g, [&](int x_cb, int parity, double *v) {
        double q;
        gauge_obs_site(a, x_cb, parity, v[0], v[1], q);
      });
      two_stage(a.volume_cb, 1, g + 4, [&](int x_cb, int parity, double *v) {
        double sp, tm;
        gauge_obs_site(a, x_cb, parity, sp, tm, v[0]);
        if (rq.density) rq.density[(size_t)parity * a.volume_cb + x_cb] = v[0];
      });
      return 0;
    }
  };
} // namespace b200

extern "C" {
int twin_gauge_flow(void *const out[4], const void *const in[4], const int X[4], int precision, const int *paths,
                    const int *length, const double *coeff, int num_paths, int max_length, double epsilon, int n_steps,
                    void *stream)
{
  return gauge_flow<FlowTwin>(out, in, X, precision, paths, length, coeff, num_paths, max_length, epsilon, n_steps, stream);
}

int twin_gauge_observables(double energy[3], double *qcharge, double *density, const void *const qdp[4], const int X[4],
                           int precision, void *stream)
{
  return gauge_observables<FlowTwin>(energy, qcharge, density, qdp, X, precision, stream);
}
}
