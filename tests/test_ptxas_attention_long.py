"""attn_long_kernel must compile to an unserialised wgmma pipeline, like the kernels tests/test_ptxas_pipeline.py names (that test matches
by substring, and "attn_kernel" does not match this kernel's name).  Besides C7510 / C7520 this fails on C7515: ptxas reports it when a
plain instruction writes an accumulator inside a pipeline stage -- what a zero-initialised O accumulator turns into here -- and it also
serialises every wgmma.  C7519 (an injected warpgroup.arrive, which the O rescale may cause) is reported but tolerated."""
import re

import test_ptxas_pipeline as tp

NAME = "attn_long_kernel"


def test_long_attention_kernel_is_in_the_build_log_and_not_serialised():
    log = tp._build_log()
    props = re.findall(r"Function properties for (\S+)", log)
    assert any(NAME in p for p in props), f"{NAME} missing from the ptxas -v output in {tp.LOG}"
    mine = [code for code, fn in tp._findings(log) if NAME in fn]
    print(f"{NAME}: {mine.count('C7519')} C7519")
    bad = sorted({c for c in mine if c in ("C7510", "C7515", "C7520")})
    assert not bad, f"ptxas serialises the wgmma of {NAME}: " + ", ".join(bad)
