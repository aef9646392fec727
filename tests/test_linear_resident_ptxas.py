"""CPU guard on the resident-weight Linear kernel: its A operands come from
registers, and ptxas serialises the MMAs when the instructions that define
those registers sit in a divergent branch (C7520), as well as for the reasons
tests/test_wgmma_ptxas.py checks (C7515 / C7517).  Reads the `-Xptxas -v` log
the library Makefile writes; skips when the library has not been built here."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "build", "csrc", "linear_tf32.ptxas.log")
KERNEL = "linear_tf32_kernel_resident"


def test_resident_kernel_mmas_not_serialised():
    if not os.path.exists(LOG):
        pytest.skip(f"ptxas log not built: {LOG}")
    text = open(LOG).read()
    assert f"Function properties for _ZN5fbbev{len(KERNEL)}{KERNEL}" in text, (
        "no resident-kernel entries in the log")
    bad = [line for line in text.splitlines()
           if re.search(r"\(C75(15|17|20)\)", line) and KERNEL in line]
    assert not bad, "\n".join(bad)
