"""CPU tier: the multi-shift CG entry point b200_invert_multishift_cg refuses null arguments and bad parameter blocks before it
needs a device, and without a GPU refuses a valid call like every compute entry point (no CPU fallback); its Python wrapper
refuses a wrong-precision field or a bad offset list before the call; and the build's machine code for the shift update
moves 16 bytes per access with no register spills in any multi-shift kernel."""
import ctypes as C
import os
import re
import shutil
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest

from quda_b200 import dirac as DR
from quda_b200 import lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "quda_b200", "csrc", "_obj")


def _dirac(lib, buf):
    """a Wilson-PC operator over host memory: creating one only records descriptors, it touches no device"""
    h = C.c_void_p()
    X = (C.c_int * 4)(4, 4, 4, 4)
    g = L.Gauge(buf.ctypes.data, 0, 1, 18, 1.0, 1.0, -1, 1, 1)
    assert lib.b200_dirac_create(C.byref(h), L.DIRAC_WILSONPC, 8, X, C.byref(g), None, None, 0.12, 0, None, None) == 0
    return h


def _param(offsets, tols=None):
    p = L.MultiShiftParam()
    p.n_shift, p.maxiter, p.delta = len(offsets), 10, 0.1
    for j, o in enumerate(offsets[:L.MAX_SHIFTS]):
        p.offset[j] = o
        p.tol_offset[j] = 1e-10 if tols is None else tols[j]
    return p


@pytest.fixture
def setup():
    lib = L.load()
    buf = np.zeros(1 << 16, dtype=np.uint8)
    xs = (L.Spinor * L.MAX_SHIFTS)(*[L.Spinor(buf.ctypes.data, None, 0, 128, 1) for _ in range(L.MAX_SHIFTS)])
    b = L.Spinor(buf.ctypes.data, None, 0, 128, 1)
    h = _dirac(lib, buf)
    yield lib, h, xs, b, buf
    lib.b200_dirac_destroy(h)


def test_multishift_refuses_null_arguments(setup):
    lib, h, xs, b, _ = setup
    p = _param([0.0, 0.1])
    assert lib.b200_invert_multishift_cg(None, None, xs, C.byref(b), C.byref(p)) == -1  # B200_ERR_INVALID
    assert b"null argument" in lib.b200_last_error()
    assert lib.b200_invert_multishift_cg(h, None, xs, C.byref(b), None) == -1
    assert b"null argument" in lib.b200_last_error()
    assert lib.b200_invert_multishift_cg(h, None, None, C.byref(b), C.byref(p)) == -1
    assert b"null spinor" in lib.b200_last_error()
    assert lib.b200_invert_multishift_cg(h, None, xs, None, C.byref(p)) == -1
    assert b"null spinor" in lib.b200_last_error()


@pytest.mark.parametrize("offsets,tols,match", [
    ([], None, b"n_shift 0"),
    ([0.01 * j for j in range(33)], None, b"n_shift 33"),
    ([0.0, 1.0, 0.5], None, b"non-decreasing"),
    ([0.0, float("nan")], None, b"not finite"),
    ([0.0, float("inf")], None, b"not finite"),
    ([0.0, 0.1], [1e-10, 0.0], b"tol_offset 1"),
    ([0.0, 0.1], [-1e-10, 1e-10], b"tol_offset 0"),
], ids=["none", "33", "unordered", "nan", "inf", "zero-tol", "negative-tol"])
def test_multishift_refuses_a_bad_parameter_block(setup, offsets, tols, match):
    lib, h, xs, b, _ = setup
    p = _param(offsets, tols)
    assert lib.b200_invert_multishift_cg(h, None, xs, C.byref(b), C.byref(p)) == -1
    assert match in lib.b200_last_error()


def test_multishift_refuses_a_missing_solution_field(setup):
    lib, h, xs, b, _ = setup
    xs[2].v = None
    p = _param([0.0, 0.1, 1.0])
    assert lib.b200_invert_multishift_cg(h, None, xs, C.byref(b), C.byref(p)) == -1
    assert b"descriptor 2" in lib.b200_last_error()


def test_multishift_refuses_without_a_gpu(setup):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lib, h, xs, b, _ = setup
    p = _param([0.0, 0.1, 1.0])
    assert lib.b200_invert_multishift_cg(h, None, xs, C.byref(b), C.byref(p)) == -4  # B200_ERR_NO_DEVICE
    assert b"no CPU path" in lib.b200_last_error()


def test_multishift_wrapper_refuses_a_precision_mismatch():
    """the C ABI reads every x_j and b in the precise operator's precision (the stand-ins have no library handle: reaching the
    call would fail differently)"""
    precise = SimpleNamespace(prec=8)
    f8, f4 = SimpleNamespace(prec=8), SimpleNamespace(prec=4)
    for xs, b in (([f8, f4], f8), ([f4, f8], f8), ([f8, f8], f4)):
        with pytest.raises(L.B200Error, match="precision"):
            DR.invert_multishift_cg(precise, None, xs, b, [0.0, 0.1])


@pytest.mark.parametrize("offsets,kw,match", [
    ([], {}, "between 1 and"),
    ([0.01 * j for j in range(33)], {}, "between 1 and"),
    ([0.1, 0.0], {}, "non-decreasing"),
    ([0.0, float("nan")], {}, "finite"),
    ([0.0, 0.1], dict(tol_offset=[1e-10]), "one positive tolerance"),
    ([0.0, 0.1], dict(tol_offset=[1e-10, 0.0]), "one positive tolerance"),
], ids=["none", "33", "unordered", "nan", "short-tol", "zero-tol"])
def test_multishift_wrapper_refuses_a_bad_offset_list(offsets, kw, match):
    precise = SimpleNamespace(prec=8)
    xs = [SimpleNamespace(prec=8) for _ in offsets]
    with pytest.raises(L.B200Error, match=match):
        DR.invert_multishift_cg(precise, None, xs, SimpleNamespace(prec=8), offsets, **kw)


_needs_obj = pytest.mark.skipif(shutil.which("cuobjdump") is None or not os.path.exists(os.path.join(OBJ, "dirac.o")),
                                reason="needs cuobjdump and the build's object files (__graft_entry__.build())")


@_needs_obj
def test_shift_update_moves_16_bytes_per_access():
    out = subprocess.run(["cuobjdump", "-sass", os.path.join(OBJ, "dirac.o")], capture_output=True, text=True,
                         errors="replace").stdout
    funs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1) if "ms_update_xp_kernel" in m.group(1) else None
            if cur:
                funs[cur] = []
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
        if m and cur:
            funs[cur].append(m.group(1))
    assert len(funs) == 2, list(funs)  # fp64 and fp32
    for name, ins in funs.items():
        # every global load is a 16-byte field access or an 8-byte read of the scalar block
        loads = [i for i in ins if re.search(r"\bLDG\.", i)]
        assert any(".128" in i for i in loads), (name, loads)
        assert all(".128" in i or "LDG.E.64.CONSTANT" in i for i in loads), (name, loads)
        stores = [i for i in ins if re.search(r"\bSTG\.", i)]
        assert stores and all(".128" in i for i in stores), (name, stores)


@_needs_obj
def test_multishift_kernels_do_not_spill():
    log = open(os.path.join(OBJ, "dirac.ptxas.log"), errors="replace").read()
    found = 0
    for m in re.finditer(r"Compiling entry function '(\S+)'.*?(\d+) bytes spill stores, (\d+) bytes spill loads", log, re.S):
        if re.search(r"ms_(dot|update_r|update_xp|replace_r)_kernel", m.group(1)):
            found += 1
            assert m.group(2) == "0" and m.group(3) == "0", m.group(1)
    assert found == 8, found
