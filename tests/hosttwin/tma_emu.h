// TEST-ONLY emulation of the TMA-staged marching kernel (quda_b200/csrc/tma_kernel.cuh) on the CPU.
//
// It runs the product's plan, tensor-map descriptions, box coordinates, per-thread shared-memory offsets, producer
// program and site arithmetic (quda_b200/csrc/tma.h) against an emulated shared memory:
//   * box loads are interpreted from the TmaDesc exactly as cuTensorMapEncodeTiled / cp.async.bulk.tensor define them
//     (dense box in dimension order, out-of-bounds elements zero-filled);
//   * producer and consumers run as two programs coupled only through ring-slot ownership (the mbarrier full / empty
//     protocol): the producer runs as far ahead as the slots allow, a slot may only be overwritten after the consumers
//     released it, released slots are poisoned, and a state in which neither side can advance is reported as a deadlock.
// What it cannot check: PTX syntax and the phase-parity arithmetic of the real mbarriers (GPU tests do).
#pragma once

#include <cmath>
#include <cstring>
#include <vector>

#include "../../quda_b200/csrc/tma.h"

namespace b200
{

  inline void tma_emu_box_load(unsigned char *dst, const TmaDesc &d, const int *c)
  {
    size_t o = 0;
    const unsigned char *base = static_cast<const unsigned char *>(d.base);
    for (unsigned i4 = 0; i4 < d.box[4]; i4++)
      for (unsigned i3 = 0; i3 < d.box[3]; i3++)
        for (unsigned i2 = 0; i2 < d.box[2]; i2++)
          for (unsigned i1 = 0; i1 < d.box[1]; i1++)
            for (unsigned i0 = 0; i0 < d.box[0]; i0++, o += 4) {
              const long long x[5] = {c[0] + (long long)i0, c[1] + (long long)i1, c[2] + (long long)i2, c[3] + (long long)i3, c[4] + (long long)i4};
              bool in = true;
              unsigned long long off = 0;
              for (int k = 0; k < 5; k++) {
                if (x[k] < 0 || (unsigned long long)x[k] >= d.dim[k]) in = false;
                off += (unsigned long long)x[k] * d.stride[k];
              }
              if (in)
                memcpy(dst + o, base + off, 4);
              else
                memset(dst + o, 0, 4);
            }
  }

  struct TmaEmuOp {
    int ring; // 0 centre, 1 halo, 2 link
    long long n;
    TmaItem it;
    int arg; // slice (centre) or d (link)
  };

  struct TmaEmuRecorder {
    std::vector<TmaEmuOp> ops;
    void center(int n, const TmaItem &it, int slice) { ops.push_back({0, n, it, slice}); }
    void halo(int n, const TmaItem &it) { ops.push_back({1, n, it, 0}); }
    void link(long long ln, const TmaItem &it, int d) { ops.push_back({2, ln, it, d}); }
    void prefetch_link(const TmaItem &, int) { n_prefetch++; } // L2 hint only: no functional effect
    long n_prefetch = 0;
  };

  // one CTA; returns 0 or an error code (message via set_error)
  template <class P, int recon, bool dagger, bool xpay, OpType op, int PD>
  int tma_emu_cta(const DslashArgs<P, recon> &arg, const TmaPlan &plan, const TmaDesc (*descs)[TM_COUNT], int cta, int n_cta, long &visited)
  {
    using real = typename P::real;
    using Raw = typename GaugeView<P, recon>::Raw;
    constexpr bool LSTREAM = PD > 0;
    int w0, w1;
    tma_work_range(w0, w1, plan, cta, n_cta);
    if (w0 >= w1) return 0;
    const int NL = plan.n_link_slots, NCS = plan.n_center_slots, NHS = plan.n_halo_slots;
    if (LSTREAM != (NL == 0)) return set_error(B200_ERR_INVALID, "emulation: link mode / plan mismatch");
    std::vector<unsigned char> smem(plan.smem_bytes, 0xA5);
    std::vector<long long> own_c(NCS, -1), own_h(NHS, -1), own_l(NL > 0 ? NL : 1, -1);
    TmaEmuRecorder rec;
    tma_producer_program(plan, w0, w1, rec);
    size_t pi = 0;

    auto poison = [&](int off, int bytes) { memset(smem.data() + off, 0xFF, bytes); }; // NaN pattern for every real type
    auto desc_of = [&](const TmaItem &it, int id) -> const TmaDesc & { return descs[plan.n_parity == 2 ? it.par : 0][id]; };
    // producer: run as far as the slot ownership allows
    auto produce = [&]() -> int {
      int done = 0;
      while (pi < rec.ops.size()) {
        const TmaEmuOp &o = rec.ops[pi];
        if (o.ring == 0) {
          const int s = (int)(o.n % NCS);
          if (own_c[s] >= 0) break;
          TmaBox b;
          tma_center_box(b, o.it, o.arg);
          const TmaDesc &d = desc_of(o.it, b.map);
          if (tma_box_bytes(d) != plan.NC * plan.srow) return set_error(B200_ERR_INVALID, "centre box bytes != expect_tx");
          tma_emu_box_load(smem.data() + plan.off_center + s * plan.center_bytes + b.dst, d, b.c);
          own_c[s] = o.n;
        } else if (o.ring == 1) {
          const int s = (int)(o.n % NHS);
          if (own_h[s] >= 0) break;
          TmaBox b[4];
          tma_halo_boxes(b, plan, o.it);
          int bytes = 0;
          for (int k = 0; k < 4; k++) {
            const TmaDesc &d = desc_of(o.it, b[k].map);
            bytes += tma_box_bytes(d);
            tma_emu_box_load(smem.data() + plan.off_halo + s * plan.halo_bytes + b[k].dst, d, b[k].c);
          }
          if (bytes != plan.NH * plan.srow) return set_error(B200_ERR_INVALID, "halo box bytes != expect_tx");
          own_h[s] = o.n;
        } else {
          const int s = (int)(o.n % NL);
          if (own_l[s] >= 0) break;
          TmaBox b[3];
          const int nb = tma_link_boxes(b, plan, o.it, o.arg);
          int bytes = 0;
          for (int k = 0; k < nb; k++) {
            const TmaDesc &d = desc_of(o.it, b[k].map);
            if (!d.valid) return set_error(B200_ERR_INVALID, "link box uses an invalid map");
            bytes += tma_box_bytes(d);
            tma_emu_box_load(smem.data() + plan.off_link + s * plan.link_bytes + b[k].dst, d, b[k].c);
          }
          if (bytes != 2 * plan.NC * plan.grow) return set_error(B200_ERR_INVALID, "link box bytes != expect_tx");
          own_l[s] = o.n;
        }
        pi++;
        done++;
      }
      return done;
    };
    // consumer-side wait: the load must be resident; otherwise let the producer run; if it cannot, that is a deadlock
    auto wait = [&](std::vector<long long> &own, int slot, long long n, const char *what) -> int {
      if (own[slot] == n) return 0;
      const int r = produce();
      if (r < 0) return r;
      if (own[slot] != n)
        return set_error(B200_ERR_INVALID, "TMA pipeline deadlock: CTA %d waits for %s load %lld (slot holds %lld, producer at op %zu/%zu)", cta,
                         what, n, own[slot], pi, rec.ops.size());
      return 0;
    };

    const int nthr = plan.n_cwarps * 32;
    std::vector<TmaThread> th(nthr);
    for (int t = 0; t < nthr; t++) tma_thread_init(th[t], plan, t);
    std::vector<real> acc((size_t)nthr * 24);
    std::vector<Raw> lk((size_t)nthr * 8); // the consumers' link registers (register-stream mode)
    std::vector<TmaSite> cur(nthr), nxt(nthr);
    // ring positions exactly as the CUDA consumers track them; cn / hn / ln are the load numbers they must hold
    TmaPos c0p {0, 0}, hp {0, 0}, lp {0, 0};
    long long cn = 0, hn = 0, ln = 0;
    {
      const int r = produce(); // the producer starts before anybody waits
      if (r < 0) return r;
    }
    TmaItem it;
    tma_item(it, plan, w0);
    for (int t = 0; t < nthr; t++) {
      tma_site(cur[t], plan, th[t], it);
      if (LSTREAM && th[t].active) {
        memset(&lk[(size_t)t * 8], 0xFF, 8 * sizeof(Raw)); // registers not loaded yet hold garbage
        if constexpr (LSTREAM) tma_load_links<P, recon, PD>(&lk[(size_t)t * 8], arg.U, cur[t]);
      }
    }
    for (int w = w0; w < w1; w++) {
      {
        TmaItem chk;
        tma_item(chk, plan, w);
        if (chk.par != it.par || chk.y0 != it.y0 || chk.z0 != it.z0 || chk.t != it.t)
          return set_error(B200_ERR_INVALID, "tma_item_next disagrees with tma_item at item %d", w);
      }
      const bool first = (w == w0) || (it.t == 0);
      const bool last = (w == w1 - 1) || (it.t == plan.T - 1);
      const bool have_next = w + 1 < w1;
      TmaItem nit = it;
      if (have_next) tma_item_next(nit, it, plan, w + 1);
      for (int t = 0; t < nthr; t++) {
        nxt[t] = cur[t];
        if (have_next) tma_site(nxt[t], plan, th[t], nit);
      }
      const TmaPos c1p = tma_pos_next(c0p, NCS), c2p = tma_pos_next(c1p, NCS);
      if (first) {
        if (int e = wait(own_c, c0p.slot, cn, "centre")) return e;
        if (int e = wait(own_c, c1p.slot, cn + 1, "centre")) return e;
      }
      if (int e = wait(own_c, c2p.slot, cn + 2, "centre")) return e;
      if (int e = wait(own_h, hp.slot, hn, "halo")) return e;
      // slices t-1 and t must still be the loads this item expects (they were waited for by earlier items)
      if (own_c[c0p.slot] != cn || own_c[c1p.slot] != cn + 1)
        return set_error(B200_ERR_INVALID, "TMA pipeline: centre slot overwritten while live (CTA %d item %d)", cta, w);
      // the phase parity the CUDA consumer waits with must be the parity of the pass that load belongs to
      if (c0p.phase != (unsigned)((cn / NCS) & 1) || c2p.phase != (unsigned)(((cn + 2) / NCS) & 1) || hp.phase != (unsigned)((hn / NHS) & 1))
        return set_error(B200_ERR_INVALID, "TMA pipeline: ring phase tracking out of step (CTA %d item %d)", cta, w);
      TmaBases b;
      b.cm = smem.data() + plan.off_center + c0p.slot * plan.center_bytes;
      b.c0 = smem.data() + plan.off_center + c1p.slot * plan.center_bytes;
      b.cp = smem.data() + plan.off_center + c2p.slot * plan.center_bytes;
      b.halo = smem.data() + plan.off_halo + hp.slot * plan.halo_bytes;
      for (size_t i = 0; i < acc.size(); i++) acc[i] = 0;
      auto dim = [&](auto D) -> int {
        constexpr int d = decltype(D)::value;
        if constexpr (LSTREAM) {
          for (int t = 0; t < nthr; t++) {
            if (!th[t].active) continue;
            tma_hop_pair_stream<P, recon, dagger, d, (PD > 0 ? PD : 1)>(&acc[(size_t)t * 24], arg.U, &lk[(size_t)t * 8], plan, th[t], b, cur[t], nxt[t], have_next);
          }
          return 0;
        } else {
          if (int e = wait(own_l, lp.slot, ln, "link")) return e;
          if (lp.phase != (unsigned)((ln / NL) & 1)) return set_error(B200_ERR_INVALID, "TMA pipeline: link ring phase out of step");
          const unsigned char *stage = smem.data() + plan.off_link + lp.slot * plan.link_bytes;
          for (int t = 0; t < nthr; t++) {
            if (!th[t].active) continue;
            tma_hop_pair<P, recon, dagger, d>(&acc[(size_t)t * 24], arg.U, plan, th[t], b, stage, cur[t]);
          }
          own_l[lp.slot] = -1; // released
          poison(plan.off_link + lp.slot * plan.link_bytes, plan.link_bytes);
          lp = tma_pos_next(lp, NL);
          ln++;
          const int r = produce(); // aggressive producer: refill as soon as a slot is free
          return r < 0 ? r : 0;
        }
      };
      if (int e = dim(std::integral_constant<int, 0> {})) return e;
      if (int e = dim(std::integral_constant<int, 1> {})) return e;
      if (int e = dim(std::integral_constant<int, 2> {})) return e;
      if (int e = dim(std::integral_constant<int, 3> {})) return e;
      auto release_c = [&](int slot) {
        own_c[slot] = -1;
        poison(plan.off_center + slot * plan.center_bytes, plan.center_bytes);
      };
      release_c(c0p.slot);
      own_h[hp.slot] = -1;
      poison(plan.off_halo + hp.slot * plan.halo_bytes, plan.halo_bytes);
      if (last) {
        release_c(c1p.slot);
        release_c(c2p.slot);
      }
      {
        const int r = produce();
        if (r < 0) return r;
      }
      for (int t = 0; t < nthr; t++) {
        if (!th[t].active) continue;
        tma_epilogue<P, recon, dagger, xpay, op>(&acc[(size_t)t * 24], arg, cur[t].x_cb, cur[t].par);
        visited++;
      }
      c0p = last ? tma_pos_next(c2p, NCS) : c1p;
      cn += last ? 3 : 1;
      hp = tma_pos_next(hp, NHS);
      hn++;
      it = nit;
      cur.swap(nxt);
    }
    if (NL > 0 && plan.l2_prefetch_items > 0 && rec.n_prefetch != 4L * ((w1 - w0) - 1))
      return set_error(B200_ERR_INVALID, "TMA pipeline: CTA %d prefetched %ld link stages for %d items", cta, rec.n_prefetch, w1 - w0);
    if (pi != rec.ops.size())
      return set_error(B200_ERR_INVALID, "TMA pipeline: CTA %d finished with %zu producer ops never issued", cta, rec.ops.size() - pi);
    return 0;
  }

  // whole launch on a grid of (at most) n_sm CTAs; kTmaSkip if the shape is not served (the caller then walks the gather
  // kernel's grid).  Which ops the kernel serves: plan.h::dispatch_tma.
  template <class P, int recon, bool dagger, bool xpay, OpType op>
  int tma_emu_launch(OpCfg<dagger, xpay, op>, const LaunchRequest &rq, const DslashArgs<P, recon> &arg, int n_sm)
  {
    TmaPlan plan;
    TmaKnobs knobs {rq.tma_ty, rq.tma_tz, rq.tma_link_slots, rq.tma_center_slots, rq.tma_halo_slots, rq.tma_l2_prefetch};
    if (!tma_make_plan<P, recon>(plan, arg.geom, arg.n_parity, arg.parity, knobs)) return kTmaSkip;
    if (plan.smem_bytes > kTmaSmemBudget) return set_error(B200_ERR_INVALID, "TMA plan needs %d bytes of shared memory", plan.smem_bytes);
    TmaDesc descs[2][TM_COUNT];
    for (int pi = 0; pi < arg.n_parity; pi++) {
      tma_make_descs(descs[pi], arg, plan, arg.n_parity == 2 ? pi : arg.parity);
      for (int k = 0; k < TM_COUNT; k++)
        if (!tma_desc_ok(descs[pi][k])) return kTmaSkip;
    }
    const int grid = tma_grid(rq, plan.n_items, n_sm);
    long visited = 0;
    int err = 0;
#pragma omp parallel for reduction(+ : visited) schedule(dynamic)
    for (int cta = 0; cta < grid; cta++) {
      long v = 0;
      int e;
      if (plan.n_link_slots > 0)
        e = tma_emu_cta<P, recon, dagger, xpay, op, 0>(arg, plan, descs, cta, grid, v);
      else if (rq.tma_prefetch == 2)
        e = tma_emu_cta<P, recon, dagger, xpay, op, 2>(arg, plan, descs, cta, grid, v);
      else if (rq.tma_prefetch == 4)
        e = tma_emu_cta<P, recon, dagger, xpay, op, 4>(arg, plan, descs, cta, grid, v);
      else
        e = tma_emu_cta<P, recon, dagger, xpay, op, 3>(arg, plan, descs, cta, grid, v);
      visited += v;
      if (e) {
#pragma omp critical
        err = e;
      }
    }
    if (err) return err;
    if (visited != (long)arg.geom.volume_cb * arg.n_parity)
      return set_error(B200_ERR_INVALID, "TMA work ranges visited %ld of %ld sites", visited, (long)arg.geom.volume_cb * arg.n_parity);
    return 0;
  }

} // namespace b200
