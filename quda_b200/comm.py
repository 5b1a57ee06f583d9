"""4-d process grid + halo exchange plumbing (one process per GPU, torch.distributed for bootstrap).

What the reference does with MPI/QMP + CUDA IPC (lib/comm_common.cpp:101-134 topology,
lib/targets/cuda/comm_target.cpp:37-167 IPC handle exchange, lib/color_spinor_field.cpp:980-1255 pack / send /
query / scatter) collapses here, on an NVSwitch box, to ONE schedule:

    pack kernel stores spin-projected faces straight into the neighbour's ghost buffer over NVLink and then
    sets an arrival flag there (release, system scope)  ->  interior kernel runs meanwhile  ->  the fused exterior
    kernel acquires the flags and finishes the boundary sites.

No host polling, no MPI in the critical path.  Modes:
  "p2p"   peer buffers mapped with CUDA IPC (b200_ipc_*); flags carry a per-exchange sequence number and the
          ghost buffers are double-buffered, so successive Dslash applications need no extra synchronisation
  "nccl"  portable fallback: pack into local send buffers, grouped ncclSend/ncclRecv via torch.distributed
  "self"  single rank that is its own neighbour (the reference's --partition trick) -- used by tests
  "host"  CPU-tier tests only: numpy buffers + gloo send/recv, compute by the host twin

Multi-RHS batches (`HaloExchange(n_src=...)`, lists of fields in `apply_wilson_distributed`): every ghost region holds one
slab per source and the whole batch travels in ONE exchange -- one pack launch and one arrival signal per face
(b200_pack_ghost_multi; reference: lib/dslash_pack2.cu:55-403), one message per face in the staged modes.
"""
import ctypes as C
import os

import numpy as np

from . import dslash as D
from . import fields as F
from . import lib as L


class ProcessGrid:
    """Lexicographic rank <-> coordinate map with t running fastest (tests/utils/host_utils.cpp:667-672)."""

    def __init__(self, dims, rank):
        self.dims = [int(d) for d in dims]
        self.size = int(np.prod(self.dims))
        self.rank = rank
        self.coords = self.coords_of(rank)

    def coords_of(self, rank):
        c = [0, 0, 0, 0]
        for d in (3, 2, 1, 0):
            c[d] = rank % self.dims[d]
            rank //= self.dims[d]
        return c

    def rank_of(self, coords):
        r = 0
        for d in range(4):
            r = r * self.dims[d] + (coords[d] % self.dims[d])
        return r

    def neighbor(self, d, direction):
        c = list(self.coords)
        c[d] += direction
        return self.rank_of(c)

    def comm_dim(self):
        return [1 if g > 1 else 0 for g in self.dims]

    def first_time_slice(self):
        return self.coords[3] == 0

    def last_time_slice(self):
        return self.coords[3] == self.dims[3] - 1

    @staticmethod
    def default_dims(world):
        """split t first, then z, then y: 2 -> (1,1,1,2), 4 -> (1,1,2,2), 8 -> (1,2,2,2)"""
        g, d = [1, 1, 1, 1], 3
        while world > 1:
            assert world % 2 == 0, "process grid helper supports power-of-two worlds"
            g[d] *= 2
            world //= 2
            d = d - 1 if d > 0 else 3
        return g


def local_slice(global_field, Xg, Xl, coords, kind):
    """Cut the local block out of a global oracle-order field.
    kind 'gauge': [4][V][...] parity-major sites; 'spinor1': single parity [Vh][...] (give parity via tuple
    ('spinor1', p)); 'spinor2': full [2*Vh][...]; 'clover': [V][...]"""
    off = [coords[d] * Xl[d] for d in range(4)]
    Vhg, Vhl = F.volume_cb(Xg), F.volume_cb(Xl)

    def site_map(parity):
        c = F.cb_coords(Xl, parity) + np.array(off)
        return F.cb_index(c, Xg)

    if kind == "gauge":
        g = np.asarray(global_field).reshape((4, 2, Vhg) + global_field.shape[2:])
        return np.ascontiguousarray(np.stack([g[:, p, site_map(p)] for p in range(2)], axis=1)).reshape(
            (4, 2 * Vhl) + global_field.shape[2:])
    if kind == "clover":
        c = np.asarray(global_field).reshape((2, Vhg) + global_field.shape[1:])
        return np.ascontiguousarray(np.stack([c[p, site_map(p)] for p in range(2)])).reshape(
            (2 * Vhl,) + global_field.shape[1:])
    if kind == "spinor2":
        s = np.asarray(global_field).reshape((2, Vhg) + global_field.shape[1:])
        return np.ascontiguousarray(np.stack([s[p, site_map(p)] for p in range(2)])).reshape(
            (2 * Vhl,) + global_field.shape[1:])
    if isinstance(kind, tuple) and kind[0] == "spinor1":
        return np.ascontiguousarray(np.asarray(global_field)[site_map(kind[1])])
    raise ValueError(kind)


def _lex_of_sites(X):
    """lexicographic index ((t X2 + z) X1 + y) X0 + x of every parity-major QDP site"""
    c = np.concatenate([F.cb_coords(X, p) for p in range(2)])
    return ((c[:, 3] * X[2] + c[:, 2]) * X[1] + c[:, 1]) * X[0] + c[:, 0]


def extend_gauge(grid, gauge_local, X, dist):
    """The local QDP-order links ([4][V][3][3][2], numpy or torch) extended by a depth-1 halo in every partitioned dimension
    of `grid`: QDP order on X_e = X + 2 comm_dim (parity of the extended coordinates), the lattice the clover kernels read
    with border = comm_dim (createExtendedGauge with R = 1, lib/gauge_field.cpp / lib/copy_gauge_extended.cu).  Dimension by
    dimension, each rank sends its first and last interior slabs of the already-extended array to its neighbours, so the
    halos of earlier dimensions travel along and corners arrive.  torch.distributed send / recv: gloo on the host, NCCL on
    GPUs (tensors on the device).  Returns the same kind of array as it was given."""
    import torch
    is_np = isinstance(gauge_local, np.ndarray)
    g = torch.from_numpy(np.ascontiguousarray(gauge_local)) if is_np else gauge_local
    X = [int(v) for v in X]
    border = grid.comm_dim()
    Xe = [X[d] + 2 * border[d] for d in range(4)]
    tail = tuple(g.shape[2:])
    lex = torch.empty((4, X[0] * X[1] * X[2] * X[3]) + tail, dtype=g.dtype, device=g.device)
    lex[:, torch.from_numpy(_lex_of_sites(X)).to(g.device)] = g
    ext = torch.zeros((4, Xe[3], Xe[2], Xe[1], Xe[0]) + tail, dtype=g.dtype, device=g.device)
    ext[:, border[3]:border[3] + X[3], border[2]:border[2] + X[2], border[1]:border[1] + X[1], border[0]:border[0] + X[0]] = \
        lex.reshape((4, X[3], X[2], X[1], X[0]) + tail)
    for d in range(4):
        if not border[d]:
            continue
        ax = 4 - d
        lo, hi = ext.narrow(ax, 1, 1).contiguous(), ext.narrow(ax, X[d], 1).contiguous()
        into_hi, into_lo = torch.empty_like(lo), torch.empty_like(hi)
        bwd, fwd = grid.neighbor(d, -1), grid.neighbor(d, +1)
        # my first slab is the backward neighbour's upper halo, my last one the forward neighbour's lower halo; with the
        # same peer on both sides, the sends and the receives pair up in posting order
        ops = [dist.P2POp(dist.isend, lo, bwd, tag=2 * d), dist.P2POp(dist.isend, hi, fwd, tag=2 * d + 1),
               dist.P2POp(dist.irecv, into_hi, fwd, tag=2 * d), dist.P2POp(dist.irecv, into_lo, bwd, tag=2 * d + 1)]
        for req in dist.batch_isend_irecv(ops):
            req.wait()
        ext.narrow(ax, Xe[d] - 1, 1).copy_(into_hi)
        ext.narrow(ax, 0, 1).copy_(into_lo)
    out = ext.reshape((4, Xe[0] * Xe[1] * Xe[2] * Xe[3]) + tail)[:, torch.from_numpy(_lex_of_sites(Xe)).to(g.device)]
    return out.contiguous().numpy() if is_np else out.contiguous()


class HaloExchange:
    """Ghost buffers + neighbour wiring for one (lattice, precision, site-subset).  Owns its buffers (allocated once,
    like the reference's static ghost buffers, lib/lattice_field.cpp:274-303)."""

    def __init__(self, grid, X, prec, n_parity=1, mode="p2p", backend=None, dist=None, self_dims=None, n_src=1):
        self.grid, self.X, self.prec, self.n_parity, self.mode = grid, [int(v) for v in X], prec, n_parity, mode
        self.backend, self.dist = backend, dist
        # n_src > 1: every ghost region holds n_src slabs (one per source of a multi-RHS batch, src_stride[d] bytes apart) so
        # that the faces of a whole batch travel in ONE pack launch / ONE exchange with ONE arrival signal per face
        self.n_src = int(n_src)
        if not 1 <= self.n_src <= L.MAX_MULTI_RHS:
            raise L.B200Error(f"n_src {n_src} not in [1, {L.MAX_MULTI_RHS}]")
        # "self": a single rank that is its own neighbour in the dimensions of `self_dims` (default: all four)
        self.comm_dim = grid.comm_dim() if mode != "self" else [int(bool(v)) for v in (self_dims or (1, 1, 1, 1))]
        self._comm_struct = None
        self._seq = 0
        self.face_bytes = [n_parity * F.ghost_parity_bytes(X, prec, d) for d in range(4)]
        # slab layout: [buf 0|1][d][dir] ghost regions (256-byte aligned), then flags[2][4][2] (u32), counters[8], timeout
        self.src_stride = [(fb + 255) // 256 * 256 for fb in self.face_bytes]
        self.off = {}
        o = 0
        for b in range(2):
            for d in range(4):
                for dr in range(2):
                    self.off[(b, d, dr)] = o
                    o += self.n_src * self.src_stride[d] if self.comm_dim[d] else 0
        self.flag_off = o
        o += 2 * 8 * 4
        self.counter_off = o
        o += 8 * 4
        self.timeout_off = o
        o += 64
        self.mailbox_off = (o + 255) // 256 * 256   # NVLink all-reduce mailboxes (b200_comm::reduce_peer)
        o = self.mailbox_off + L.REDUCE_MAILBOX_BYTES
        self.slab_bytes = (o + 255) // 256 * 256
        # solver scalars: "callback" = torch.distributed all-reduce from the host (validated default);
        # "nvlink" = the mailbox kernel over peer memory (needs every rank mapped, world <= 16)
        # solver scalars: "nvlink" = device-side all-reduce through peer-mapped mailboxes inside the reduction kernels (no
        # host round trip); "callback" = torch.distributed all_reduce from the host (two stream syncs per CG iteration)
        self.allreduce_mode = os.environ.get("B200_ALLREDUCE", "nvlink")
        self.send_off = None
        if mode in ("p2p", "self"):
            self._init_device_slab()
        elif mode == "nccl":
            self._init_nccl()
        elif mode == "host":
            self.slab = np.zeros(self.slab_bytes, dtype=np.uint8)
            self.base = self.slab.ctypes.data
            self.send = np.zeros(self.slab_bytes, dtype=np.uint8)
        else:
            raise ValueError(mode)

    # ------------------------------------------------------------------ set-up
    def _init_device_slab(self):
        lib = L.load()
        p = C.c_void_p()
        L.check(lib.b200_comm_alloc(C.byref(p), self.slab_bytes))
        self.base = p.value
        self.peer = {self.grid.rank: self.base}
        if self.mode == "self":
            return
        h = C.create_string_buffer(64)
        L.check(lib.b200_ipc_get_handle(self.base, h))
        handles = [None] * self.grid.size
        self.dist.all_gather_object(handles, bytes(h.raw))
        need = set()
        for d in range(4):
            if self.comm_dim[d]:
                need.add(self.grid.neighbor(d, +1))
                need.add(self.grid.neighbor(d, -1))
        if self.allreduce_mode == "nvlink":
            if self.grid.size > L.MAX_RANKS:
                raise L.B200Error(f"B200_ALLREDUCE=nvlink supports up to {L.MAX_RANKS} ranks")
            need.update(range(self.grid.size))
        for r in need:
            if r == self.grid.rank:
                continue
            q = C.c_void_p()
            L.check(lib.b200_ipc_open_handle(handles[r], C.byref(q)))
            self.peer[r] = q.value
        self.dist.barrier()

    def _init_nccl(self):
        import torch
        self.slab = torch.zeros(self.slab_bytes, dtype=torch.uint8, device="cuda")
        self.send = torch.zeros(self.slab_bytes, dtype=torch.uint8, device="cuda")
        self.base = self.slab.data_ptr()

    # The exchange counter is ONE number shared by every layer that drives this exchange: once a b200_comm block exists
    # (comm_struct()), the C++ operators advance its `seq` field in place and the Python-level schedule reads / advances the
    # very same field, so mixing Dirac objects with apply_wilson_distributed can never reuse a sequence number.
    @property
    def seq(self):
        return int(self._comm_struct.seq) if self._comm_struct is not None else self._seq

    @seq.setter
    def seq(self, v):
        if self._comm_struct is not None:
            self._comm_struct.seq = int(v)
        else:
            self._seq = int(v)

    def pack_stream(self, stream=None):
        """side stream on which the pack kernel runs concurrently with the interior kernel"""
        if getattr(self, "_pack_stream", None) is None:
            import torch
            self._pack_stream = torch.cuda.Stream(priority=-1)  # high priority: never starved by spinning boundary CTAs
        return self._pack_stream

    # ------------------------------------------------------------------ per-application calls
    def start(self, in_field, in_parity, dagger, stream=None, parity_slot=0):
        """Pack the faces of `in_field` (sites of parity `in_parity`) and ship them to the neighbours.  A list of fields
        (at most `n_src`) is one batched exchange: one pack launch, one signal per face; source s lands in slab s."""
        batch = list(in_field) if isinstance(in_field, (list, tuple)) else None
        if batch is not None:
            if not 1 <= len(batch) <= self.n_src:
                raise L.B200Error(f"batch of {len(batch)} sources on an exchange created for n_src={self.n_src}")
            in_field = batch[0]
        self.seq += 1
        b = self.seq & 1
        g = self.grid
        pslot = parity_slot * F.ghost_parity_bytes(self.X, self.prec, 0)  # recomputed per d below
        if self.mode in ("p2p", "self"):
            a = L.PackArgs()
            a.abi_version, a.precision = L.ABI_VERSION, self.prec
            for d in range(4):
                a.X[d] = self.X[d]
                a.comm_dim[d] = self.comm_dim[d]
                if not self.comm_dim[d]:
                    continue
                pslot = parity_slot * F.ghost_parity_bytes(self.X, self.prec, d)
                back = self.peer[g.neighbor(d, -1)] if self.mode == "p2p" else self.base
                fwd = self.peer[g.neighbor(d, +1)] if self.mode == "p2p" else self.base
                # our low face -> backward neighbour's "from forward" slot; our high face -> forward neighbour's "from backward" slot
                a.dst[d][0] = back + self.off[(b, d, 1)] + pslot
                a.dst[d][1] = fwd + self.off[(b, d, 0)] + pslot
                a.signal[d][0] = back + self.flag_off + ((b * 4 + d) * 2 + 1) * 4
                a.signal[d][1] = fwd + self.flag_off + ((b * 4 + d) * 2 + 0) * 4
            a.block_counter = self.base + self.counter_off
            a.seq = self.seq
            a.parity, a.dagger = in_parity, int(bool(dagger))
            a.in_ = in_field.desc()
            a.stream = stream
            be = self.backend or D.cuda_backend()
            if batch is None:
                be.call("pack_ghost", C.byref(a))
            else:
                srcs = (L.Spinor * len(batch))(*[f.desc() for f in batch])
                stride = (C.c_size_t * 4)(*self.src_stride)
                be.call("pack_ghost_multi", C.byref(a), len(batch), srcs, stride)
            return
        # staged modes: pack locally (every source into its slab), then ONE exchange of the whole batch
        for s, f_in in enumerate(batch or [in_field]):
            dst = [[None, None] for _ in range(4)]
            for d in range(4):
                if self.comm_dim[d]:
                    for f in range(2):
                        dst[d][f] = self.send[self.off[(b, d, f)] + s * self.src_stride[d]:]
            D.PackGhost(dst, f_in, in_parity, dagger, self.comm_dim, stream=stream, backend=self.backend)
        m = len(batch) if batch is not None else 1
        if self.mode == "nccl":
            self._exchange_nccl(b, m)
        else:
            self._exchange_host(b, m)

    def _exchange_nccl(self, b, m=1):
        import torch.distributed as dist
        ops = []
        g = self.grid
        for d in range(4):
            if not self.comm_dim[d]:
                continue
            n = self.face_bytes[d] + (m - 1) * self.src_stride[d]
            lo, hi = self.off[(b, d, 0)], self.off[(b, d, 1)]
            # send low face backwards (arrives in their slot 1), high face forwards (arrives in their slot 0)
            ops.append(dist.P2POp(dist.isend, self.send[lo:lo + n], g.neighbor(d, -1)))
            ops.append(dist.P2POp(dist.isend, self.send[hi:hi + n], g.neighbor(d, +1)))
            ops.append(dist.P2POp(dist.irecv, self.slab[hi:hi + n], g.neighbor(d, +1)))
            ops.append(dist.P2POp(dist.irecv, self.slab[lo:lo + n], g.neighbor(d, -1)))
        for w in dist.batch_isend_irecv(ops):
            w.wait()

    def _exchange_host(self, b, m=1):
        import torch
        dist = self.dist
        g = self.grid
        for d in range(4):
            if not self.comm_dim[d]:
                continue
            n = self.face_bytes[d] + (m - 1) * self.src_stride[d]
            lo, hi = self.off[(b, d, 0)], self.off[(b, d, 1)]
            s_lo, s_hi = torch.from_numpy(self.send[lo:lo + n]), torch.from_numpy(self.send[hi:hi + n])
            r_lo, r_hi = torch.from_numpy(self.slab[lo:lo + n]), torch.from_numpy(self.slab[hi:hi + n])
            reqs = [dist.isend(s_lo, g.neighbor(d, -1), tag=2 * d), dist.isend(s_hi, g.neighbor(d, +1), tag=2 * d + 1),
                    dist.irecv(r_hi, g.neighbor(d, +1), tag=2 * d), dist.irecv(r_lo, g.neighbor(d, -1), tag=2 * d + 1)]
            for r in reqs:
                r.wait()

    def halo(self, src=0):
        """b200_halo descriptor for the exchange started last (`src`: which source of a batched exchange; all sources share
        the arrival flags and the sequence number)."""
        b = self.seq & 1
        h = L.Halo()
        for d in range(4):
            h.comm_dim[d] = self.comm_dim[d]
            for dr in range(2):
                if self.comm_dim[d]:
                    h.ghost[d][dr] = self.base + self.off[(b, d, dr)] + src * self.src_stride[d]
                    if self.mode in ("p2p", "self"):
                        h.wait_flag[d][dr] = self.base + self.flag_off + ((b * 4 + d) * 2 + dr) * 4
            h.src_stride[d] = self.src_stride[d] if self.n_src > 1 else 0
        h.seq = self.seq
        h.timeout_flag = (self.base + self.timeout_off) if self.mode in ("p2p", "self") else None
        return h

    def comm_struct(self):
        """b200_comm block for the C++ operator / solver layer (quda_b200/csrc/host/dirac.h::CommContext): peer
        destinations + signals for both ghost buffers, local receive slots + flags, and an allreduce callback for the
        solver's scalars.  The returned object must be kept alive as long as operators created with it exist."""
        assert self.mode in ("p2p", "self")
        c = L.Comm()
        g = self.grid
        for d in range(4):
            c.comm_dim[d] = self.comm_dim[d]
            if not self.comm_dim[d]:
                continue
            back = self.peer[g.neighbor(d, -1)] if self.mode == "p2p" else self.base
            fwd = self.peer[g.neighbor(d, +1)] if self.mode == "p2p" else self.base
            for b in range(2):
                c.send_dst[b][d][0] = back + self.off[(b, d, 1)]
                c.send_dst[b][d][1] = fwd + self.off[(b, d, 0)]
                c.send_signal[b][d][0] = back + self.flag_off + ((b * 4 + d) * 2 + 1) * 4
                c.send_signal[b][d][1] = fwd + self.flag_off + ((b * 4 + d) * 2 + 0) * 4
                for dr in range(2):
                    c.recv[b][d][dr] = self.base + self.off[(b, d, dr)]
                    c.recv_flag[b][d][dr] = self.base + self.flag_off + ((b * 4 + d) * 2 + dr) * 4
        c.block_counter = self.base + self.counter_off
        c.timeout_flag = self.base + self.timeout_off
        c.seq = self.seq
        if self._comm_struct is not None:
            c.reduce_seq = self._comm_struct.reduce_seq
        if self.mode == "p2p":
            c.pack_stream = self.pack_stream().cuda_stream
        if self.mode == "p2p" and g.size > 1:
            import torch
            dist = self.dist

            def _allreduce(ptr, n, _user):
                t = torch.tensor([ptr[i] for i in range(n)], dtype=torch.float64, device="cuda")
                dist.all_reduce(t)
                v = t.cpu().tolist()
                for i in range(n):
                    ptr[i] = v[i]

            self._allreduce_cb = L.ALLREDUCE_FN(_allreduce)  # keep the callback object alive
            c.allreduce_sum = C.cast(self._allreduce_cb, C.c_void_p)
            if self.allreduce_mode == "nvlink":
                c.rank, c.n_ranks = g.rank, g.size
                for r in range(g.size):
                    c.reduce_peer[r] = self.peer[r] + self.mailbox_off
        self._comm_struct = c
        return c

    def timed_out(self):
        """True if an exterior kernel gave up waiting for a neighbour (device flag set by wait_for_halo)."""
        if self.mode not in ("p2p", "self"):
            return False
        v = C.c_int(0)
        L.check(L.load().b200_comm_copy(C.byref(v), self.base + self.timeout_off, 4))
        return v.value != 0


class _RawHalo:
    """adapter so dslash._apply can take a ready-made L.Halo"""

    def __init__(self, h):
        self.h = h

    def desc(self, comm_override=None):
        if comm_override is not None:
            for d in range(4):
                if not comm_override[d]:
                    self.h.comm_dim[d] = 0
        return self.h


def apply_wilson_distributed(ex, out, in_, U, a, x, parity, dagger, op=L.OP_WILSON, A=None, stream=None, tile=None):
    """One partitioned Dslash: exchange faces of `in_` (parity 1-parity) and apply the operator.

    Schedule (device side only, nothing is polled on the host):
      side stream : pack_kernel (faces + arrival flags into the neighbours' ghost slabs over NVLink)
                    -> boundary tiles (acquire the neighbours' flags, then complete site updates)
      main stream : interior tiles (no dependence on the halo), concurrently
    The side stream forks from the main stream (so `in_` is complete) and joins it again afterwards (so `out` is
    complete and nothing that follows can overwrite `in_` while it is still being packed)."""
    multi = isinstance(out, (list, tuple))
    if multi:
        # the reference's cvector_ref batch on a partitioned lattice (lib/dslash_pack2.cu packs all sources in one launch):
        # ONE batched exchange (needs HaloExchange(n_src >= len(batch))), then b200_dslash_apply_multi runs every source on
        # its own ghost slab (halo.src_stride) behind the shared arrival counters
        if len(in_) != len(out) or (x is not None and len(x) != len(out)):
            raise L.B200Error("multi-RHS: out / in / x batches differ in length")
        out, in_, x = list(out), list(in_), (list(x) if x is not None else None)
    if any(f.n_parity != 1 for f in (in_ if multi else [in_])):
        raise NotImplementedError("full-field halo exchange: pack each parity into its slot")
    side = ex.pack_stream(stream) if ex.mode == "p2p" else None
    if side is None:
        ex.start(in_, 1 - parity, dagger, stream=stream)
        D._apply(op, out, in_, U, a, x, parity, dagger, None, A=A, halo=_RawHalo(ex.halo()), stream=stream, tile=tile,
                 backend=ex.backend)
        return
    import torch
    main = torch.cuda.current_stream() if stream is None else torch.cuda.ExternalStream(stream)
    side.wait_stream(main)
    ex.start(in_, 1 - parity, dagger, stream=side.cuda_stream)
    halo = ex.halo()
    # side stream: pack -> boundary tiles (wait for the neighbours' flags, complete updates); main stream: interior tiles
    D._apply(op, out, in_, U, a, x, parity, dagger, None, A=A, halo=_RawHalo(halo), stream=side.cuda_stream, tile=tile,
             kernel=L.KERNEL_BOUNDARY_TILES, backend=ex.backend)
    D._apply(op, out, in_, U, a, x, parity, dagger, None, A=A, halo=_RawHalo(halo), stream=main.cuda_stream, tile=tile,
             kernel=L.KERNEL_INTERIOR_TILES, backend=ex.backend)
    main.wait_stream(side)
