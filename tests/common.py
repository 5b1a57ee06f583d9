"""Shared helpers for the parity tests: build native fields from oracle-order data, run an operator through a
backend (CUDA library on the GPU tier, host twin of the same site code on the CPU tier) and compare with the
oracle using the reference's own metric."""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle
from quda_b200 import dslash as D
from quda_b200 import fields as F
from quda_b200 import lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TWIN_DIR = os.path.join(ROOT, "tests", "hosttwin")
PREC_NAME = {8: "double", 4: "single", 2: "half"}

_twin = None


def twin_backend():
    """CPU build of the product's site functions (tests/hosttwin) -- CPU-tier checker only."""
    global _twin
    if _twin is None:
        subprocess.check_call(["make", "-s", "-C", TWIN_DIR])
        # B200_TWIN_LIB: another build of the same source, e.g. `make -C tests/hosttwin asan` + LD_PRELOAD=libasan.so
        lib = C.CDLL(os.environ.get("B200_TWIN_LIB") or os.path.join(TWIN_DIR, "_build", "libhosttwin.so"))
        L.declare(lib, "twin")
        _twin = D.Backend(lib, "twin")
    return _twin


class HostMem:
    """numpy-backed buffers for the host twin"""
    @staticmethod
    def put(buf):
        return np.ascontiguousarray(buf)

    @staticmethod
    def empty(nbytes):
        return np.zeros(nbytes, dtype=np.uint8)

    @staticmethod
    def get(buf):
        return np.asarray(buf)

    @staticmethod
    def sync():
        pass


class CudaMem:
    """torch-allocated device buffers for libquda_b200.so"""
    @staticmethod
    def put(buf):
        import torch
        return torch.from_numpy(np.ascontiguousarray(buf)).cuda()

    @staticmethod
    def empty(nbytes):
        import torch
        return torch.zeros(nbytes, dtype=torch.uint8, device="cuda")

    @staticmethod
    def get(buf):
        return buf.cpu().numpy()

    @staticmethod
    def sync():
        import torch
        torch.cuda.synchronize()


class Problem:
    """Random gauge (+clover) and spinor fields in oracle order plus their native images for one (prec, recon)."""

    def __init__(self, X, prec, recon, mem, seed=137, anisotropy=1.0, antiperiodic_t=True, clover=False,
                 compressed=True, dynamic=True, host_prec=None):
        self.X, self.prec, self.recon, self.mem = [int(v) for v in X], prec, recon, mem
        self.Vh = F.volume_cb(X)
        hp = host_prec or (8 if prec == 8 else 4)
        self.hp = hp
        self.gauge = oracle.random_gauge(X, hp, seed=seed, anisotropy=anisotropy, antiperiodic_t=antiperiodic_t)
        gbuf, gmeta = F.gauge_to_native(self.gauge, X, prec, recon)
        self.U = D.GaugeField(mem.put(gbuf), X, prec, recon, gmeta, anisotropy=anisotropy,
                              t_boundary=-1 if antiperiodic_t else 1)
        self.clover = self.clover_inv = self.A = self.Ainv = None
        self.dynamic = dynamic
        if clover:
            self.clover = oracle.random_clover(X, hp, seed=seed + 1)
            self.clover_inv = oracle.clover_invert(self.clover)
            cbuf, cmeta = F.clover_to_native(self.clover, X, prec, compressed=compressed)
            self.A = D.CloverField(mem.put(cbuf), X, prec, cmeta, dynamic=dynamic)
            if not dynamic:
                ibuf, imeta = F.clover_to_native(self.clover_inv, X, prec, compressed=False)
                # static inverse field: A^{-1}/2 stored such that toNonRel(Ainv_stored toRel x) = A^{-1} x
                self.Ainv = D.CloverField(mem.put(ibuf), X, prec, imeta, dynamic=False)

    def spinor(self, seed=137, nparity=1):
        return oracle.random_spinor(self.X, self.hp, seed=seed, nparity=nparity)

    def to_dev(self, host, nparity=1):
        if nparity == 1:
            buf = F.spinor_to_native(host, self.prec)
        else:
            buf = np.concatenate([F.spinor_to_native(host[p * self.Vh:(p + 1) * self.Vh], self.prec) for p in range(2)])
        return D.ColorSpinorField(self.mem.put(buf), self.X, self.prec, nparity)

    def empty(self, nparity=1):
        return D.ColorSpinorField(self.mem.empty(nparity * F.spinor_bytes(self.X, self.prec)), self.X, self.prec, nparity)

    def to_host(self, field):
        self.mem.sync()
        raw = self.mem.get(field.buf)
        pb = F.spinor_bytes(self.X, self.prec)
        parts = [F.spinor_from_native(raw[p * pb:(p + 1) * pb], self.Vh, self.prec) for p in range(field.n_parity)]
        return np.concatenate(parts)


def assert_close(ref, test, prec, recon=18, what=""):
    lvl, dev, fails = oracle.compare_spinor(ref, test)
    tol = oracle.tolerance(PREC_NAME[prec], recon)
    assert dev <= tol, f"{what}: deviation {dev:g} > tolerance {tol:g} (prec {prec}, recon {recon}); fails={fails[:8]}"
    return dev


def host_self_exchange(X, prec, self_dims, n_src=1):
    """CPU stand-in for HaloExchange(mode="self") (one rank that is its own neighbour, arrival counters and all): the slab
    lives in numpy memory and the host twin executes the calls.  Exercises the very same Python schedule, pointer
    arithmetic and counter protocol the GPU path uses, minus the hardware."""
    from quda_b200 import comm

    class _HostSelf(comm.HaloExchange):
        def _init_device_slab(self):
            self.slab = np.zeros(self.slab_bytes, dtype=np.uint8)
            self.base = self.slab.ctypes.data
            self.peer = {self.grid.rank: self.base}

        def timed_out(self):
            return bool(self.slab[self.timeout_off:self.timeout_off + 4].view(np.int32)[0])

    return _HostSelf(comm.ProcessGrid((1, 1, 1, 1), 0), X, prec, mode="self", backend=twin_backend(), self_dims=self_dims, n_src=n_src)
