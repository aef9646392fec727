"""CPU guard on the compiled tensor-core kernels: ptxas must neither serialise
the wgmma's of `linear_tf32_kernel` / `ffn_tf32_kernel` (C7515), nor inject
warpgroup waits into them (C7517), nor spill their registers.  Reads the
`-Xptxas -v` logs the library Makefile writes next to the objects; skips when
the library has not been built here."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOGS = [os.path.join(ROOT, "build", "csrc", f"{name}.ptxas.log")
        for name in ("linear_tf32", "ffn_tf32")]
KERNELS = ("linear_tf32_kernel", "ffn_tf32_kernel")


def _read_logs():
    missing = [p for p in LOGS if not os.path.exists(p)]
    if missing:
        pytest.skip(f"ptxas logs not built: {missing}")
    return {p: open(p).read() for p in LOGS}


def test_wgmma_kernels_not_serialised():
    for path, text in _read_logs().items():
        bad = [line for line in text.splitlines()
               if re.search(r"\(C751[57]\)", line)
               and any(k in line for k in KERNELS)]
        assert not bad, f"{os.path.basename(path)}:\n" + "\n".join(bad)


def test_wgmma_kernels_do_not_spill():
    for path, text in _read_logs().items():
        seen = 0
        fn = None
        for line in text.splitlines():
            m = re.search(r"Function properties for (\S+)", line)
            if m:
                fn = m.group(1)
                continue
            m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
            if m and fn and any(k in fn for k in KERNELS):
                seen += 1
                assert (int(m.group(1)), int(m.group(2))) == (0, 0), (
                    f"{fn} spills: {line.strip()}")
            fn = None if m else fn
        assert seen > 0, f"no kernel entries found in {path}"
