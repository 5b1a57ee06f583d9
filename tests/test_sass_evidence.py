"""CPU tier: static evidence in the shipped machine code (cuobjdump on the build's sm_90a objects; nothing is executed).
  * the TMA-staged kernel really is one: UTMALDG (cp.async.bulk.tensor box loads), SYNCS.* (mbarrier arrive / expect-tx /
    try-wait) and ELECT (one elected lane of the converged producer warp) -- the mnemonics B200_PROFILING.md names;
  * the halo pack publishes arrival with system-scope ordering (MEMBAR.*.SYS before the ticket, a .SYS store for the count),
    and the boundary role acquires with a system-scope load;
  * the default fp32 kernels carry no tensor-core or TMA instructions by accident (they are plain LDG + FFMA register math)."""
import functools
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "quda_b200", "csrc", "_obj")

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None or not os.path.exists(os.path.join(OBJ, "inst_f32.o")),
                                reason="needs cuobjdump and the build's object files (__graft_entry__.build())")


@functools.lru_cache(maxsize=None)
def _dump(obj):
    return subprocess.run(["cuobjdump", "-sass", os.path.join(OBJ, obj)], capture_output=True, text=True, errors="replace").stdout


def _sass(obj, fun_regex=None):
    """{function: [instruction text]} of one object file"""
    out = _dump(obj)
    funs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1) if (fun_regex is None or re.search(fun_regex, m.group(1))) else None
            if cur:
                funs[cur] = []
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
        if m and cur:
            funs[cur].append(m.group(1))
    return funs


def test_tma_kernel_uses_tma_and_mbarriers():
    funs = _sass("inst_tma_f32.o", "dslash_tma_kernel")
    assert len(funs) >= 100
    for name, ins in funs.items():
        text = "\n".join(ins)
        assert "UTMALDG.5D" in text, name
        assert "SYNCS.ARRIVE.TRANS64" in text and "SYNCS.PHASECHK.TRANS64.TRYWAIT" in text, name
        assert "ELECT" in text, name


def test_pack_kernels_publish_and_boundary_acquires_at_system_scope():
    funs = _sass("inst_f32.o", "pack_kernel|pack_multi_kernel|dslash_boundary_kernel")
    packs = [n for n in funs if "pack_" in n]
    assert len(packs) == 2
    for n in packs:
        text = "\n".join(funs[n])
        assert text.count("MEMBAR.SC.SYS") + text.count("MEMBAR.ALL.SYS") >= 2, n   # fence before the ticket, fence before the count
        assert re.search(r"STG?\.E\S*\.SYS", text), n                                  # the arrival count: a system-scope store
        assert "ATOMG" in text or "ATOM" in text, n                                   # the local ticket
    bnd = [n for n in funs if "dslash_boundary_kernel" in n]
    assert len(bnd) == 45
    for n in bnd:
        assert re.search(r"LDG?\.E\S*\.SYS", "\n".join(funs[n])), n                       # ld.acquire.sys on the arrival counters


def test_default_kernels_are_plain_simt():
    funs = _sass("inst_f32.o", "dslash_interior_kernel")
    assert len(funs) == 96
    for name, ins in funs.items():
        text = "\n".join(ins)
        assert "FFMA" in text and "LDG" in text, name
        for bad in ("UTMALDG", "UTCMMA", "HMMA", "SYNCS"):
            assert bad not in text, (name, bad)
