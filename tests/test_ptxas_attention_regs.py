"""The fused attention kernel's consumer warpgroups must run on the 232 registers setmaxnreg gives them, not spill.

attn_kernel runs 384 threads: two consumer warpgroups and a producer warpgroup.  A block of that size starts at 168 registers per thread;
the producer warpgroup drops to 40 (setmaxnreg.dec) and the consumers rise to 232 (setmaxnreg.inc), which holds the 128-float S row block
of 256 keys and the 128-float O block of 256 channels.  This reads lib/build.log (ptxas -v, building first if needed: nvcc needs no GPU)
and the SASS of the built library (cuobjdump) and checks that every attn_kernel<LT, DN> instantiation
  * carries both register moves (USETMAXREG),
  * reports no spill stores or loads and no stack frame,
  * draws none of the wgmma pipeline warnings C7510 / C7515 / C7519 / C7520.
"""
import os
import re
import shutil
import subprocess

import pytest

from test_ptxas_pipeline import LOG, PKG, _build_log

INSTANTIATIONS = {(lt, dn) for lt in (128, 256) for dn in (64, 128, 256)}


def _attn_kernels(log):
    """{(LT, DN): (stack bytes, spill store bytes, spill load bytes)} from the ptxas -v report of every attn_kernel instantiation."""
    out, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            k = re.search(r"attn_kernelILi(\d+)ELi(\d+)E", m.group(1))
            cur = (int(k.group(1)), int(k.group(2))) if k else None
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur is not None:
            out[cur] = tuple(int(x) for x in m.groups())
            cur = None
    return out


def test_every_instantiation_is_reported():
    assert set(_attn_kernels(_build_log())) == INSTANTIATIONS, f"attn_kernel instantiations in {LOG} changed"


def test_attention_kernel_does_not_spill():
    got = _attn_kernels(_build_log())
    bad = {k: v for k, v in got.items() if v != (0, 0, 0)}
    assert not bad, "(stack, spill stores, spill loads) bytes: " + str(bad)


def test_no_wgmma_pipeline_warnings():
    bad = set()
    for line in _build_log().splitlines():
        m = re.search(r"\((C75(?:10|15|19|20))\).*function '([^']+)'", line)
        if m and re.search(r"attn_kernelILi", m.group(2)):
            bad.add((m.group(1), m.group(2)))
    assert not bad, "ptxas serialises or re-fences wgmma in: " + "; ".join(f"{c} {f}" for c, f in sorted(bad))


def _cuobjdump():
    for c in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump"):
        if c and os.path.exists(c):
            return c
    return None


@pytest.mark.skipif(_cuobjdump() is None, reason="cuobjdump (CUDA toolkit) not found")
def test_setmaxnreg_in_every_attention_kernel():
    _build_log()
    lib = os.path.join(PKG, "lib", "libsr3_b200.so")
    sass = subprocess.run([_cuobjdump(), "-sass", lib], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, check=True).stdout
    fns = re.split(r"\n\s*Function : ", sass)
    kernels = [f for f in fns if f.startswith("_ZN3sr311attn_kernel")]
    assert len(kernels) == len(INSTANTIATIONS)
    for f in kernels:
        name = f.split("\n", 1)[0].strip()
        assert re.search(r"USETMAXREG\.TRY_ALLOC\S*\s+\S+,\s*0xe8\b", f), f"{name}: no setmaxnreg.inc 232"
        assert re.search(r"USETMAXREG\.DEALLOC\S*\s+0x28\b", f), f"{name}: no setmaxnreg.dec 40"
