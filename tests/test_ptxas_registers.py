"""The tile kernel's consumer warpgroups must run on the 232 registers setmaxnreg gives them, not spill.

gemm_tile_kernel runs 384 threads: two consumer warpgroups and a producer warpgroup.  A block of that size starts at 168 registers per
thread; the producer warpgroup drops to 40 (setmaxnreg.dec) and the consumers rise to 232 (setmaxnreg.inc).  This reads lib/build.log
(ptxas -v, building first if needed: nvcc needs no GPU) and the SASS of the built library (cuobjdump) and checks that
  * every instantiation carries both register moves (USETMAXREG),
  * no instantiation spills more than SPILL_STORES allows it.
The bound of the instantiations the 16->128 sampling step runs is the few words ptxas parks in local memory across the register move, once
per CTA; the wide 256- and 128-column accumulators that still spill are listed with their byte counts so that any growth fails here.
"""
import os
import re
import shutil
import subprocess

import pytest

from test_ptxas_pipeline import LOG, PKG, _build_log

# ptxas -v spill store bytes per instantiation <BLOCK_N, MH[, ping-pong]> (CUDA 12.9, sm_90a)
SPILL_STORES = {
    (16, 1, False): 0, (16, 2, False): 0, (64, 1, True): 0,
    (32, 1, False): 24, (64, 1, False): 36, (64, 2, False): 24, (128, 1, False): 24,
    (64, 2, True): 296, (128, 1, True): 344, (128, 2, False): 890, (256, 1, False): 1182,
}


def _tile_kernels(log):
    """{(block_n, mh, pingpong): spill store bytes} from the ptxas -v report of every gemm_tile_kernel instantiation."""
    out, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            k = re.search(r"gemm_tile_kernelILi(\d+)ELi(\d+)ELb([01])E", m.group(1))
            cur = (int(k.group(1)), int(k.group(2)), k.group(3) == "1") if k else None
            continue
        m = re.search(r"(\d+) bytes spill stores", line)
        if m and cur is not None:
            out[cur] = int(m.group(1))
            cur = None
    return out


def test_every_instantiation_is_reported():
    assert set(_tile_kernels(_build_log())) == set(SPILL_STORES), f"gemm_tile_kernel instantiations in {LOG} changed"


def test_tile_kernel_spills_within_bounds():
    got = _tile_kernels(_build_log())
    over = {k: (v, SPILL_STORES.get(k)) for k, v in got.items() if v > SPILL_STORES.get(k, 0)}
    assert not over, "spill stores (got, allowed): " + str(over)


def _cuobjdump():
    for c in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump"):
        if c and os.path.exists(c):
            return c
    return None


@pytest.mark.skipif(_cuobjdump() is None, reason="cuobjdump (CUDA toolkit) not found")
def test_setmaxnreg_in_every_tile_kernel():
    _build_log()
    lib = os.path.join(PKG, "lib", "libsr3_b200.so")
    sass = subprocess.run([_cuobjdump(), "-sass", lib], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, check=True).stdout
    fns = re.split(r"\n\s*Function : ", sass)
    tiles = [f for f in fns if f.startswith("_ZN3sr316gemm_tile_kernel")]
    assert len(tiles) == len(SPILL_STORES)
    for f in tiles:
        name = f.split("\n", 1)[0].strip()
        assert re.search(r"USETMAXREG\.TRY_ALLOC\S*\s+\S+,\s*0xe8\b", f), f"{name}: no setmaxnreg.inc 232"
        assert re.search(r"USETMAXREG\.DEALLOC\S*\s+0x28\b", f), f"{name}: no setmaxnreg.dec 40"
