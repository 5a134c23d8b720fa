"""The tensor-core kernels must compile to an unserialised wgmma pipeline.

ptxas reports (with -Xptxas -v, which build.py always passes) when it gives up on keeping several wgmma.mma_async in flight:
  C7510  a function call (printf, a non-inlined helper) while wgmma are in flight
  C7520  a compiler-inserted warpgroup.arrive on a path ptxas thinks is divergent
  C7519  a compiler-inserted warpgroup.arrive (registers of the chain touched between two wgmma)
Any of the first two makes ptxas wait for every wgmma before issuing the next one, which costs a large share of the tensor-core rate.
This reads lib/build.log (building first if needed: nvcc needs no GPU) and fails if one of them names a hot-path kernel.
"""
import importlib.util
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "image-super-resolution-via-iterative-refinement_b200")
LOG = os.path.join(PKG, "lib", "build.log")

HOT = ("gemm_tile_kernel", "attn_kernel", "wgrad_kernel")
NO_ARRIVE = ("gemm_tile_kernel",)   # its stage chains are branch-free: not even an injected warpgroup.arrive


def _build_log():
    spec = importlib.util.spec_from_file_location("sr3_b200_build_for_ptxas_test", os.path.join(PKG, "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.build(force=False)                 # no-op when the library matches the sources; then the log is that compile's
    if not os.path.exists(LOG):
        mod.build(force=True)
    with open(LOG) as fh:
        return fh.read()


def _findings(log):
    out = []
    for line in log.splitlines():
        m = re.search(r"\((C75\d\d)\).*function '([^']+)'", line)
        if m:
            out.append((m.group(1), m.group(2)))
    return out


def test_build_log_covers_hot_kernels():
    log = _build_log()
    props = re.findall(r"Function properties for (\S+)", log)
    for name in HOT:
        assert any(name in p for p in props), f"{name} missing from the ptxas -v output in {LOG}"


def test_no_serialised_wgmma_in_hot_kernels():
    bad = []
    for code, fn in _findings(_build_log()):
        if code in ("C7510", "C7520") and any(h in fn for h in HOT):
            bad.append((code, fn))
        elif code == "C7519" and any(h in fn for h in NO_ARRIVE):
            bad.append((code, fn))
    assert not bad, "ptxas serialises or re-fences wgmma in: " + "; ".join(f"{c} {f}" for c, f in sorted(set(bad)))
