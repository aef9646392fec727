"""CPU guard on the fused FFN kernel's resources, from the `-Xptxas -v` log the
library Makefile writes next to the object (skips when the library has not
been built here): every `ffn_tf32_kernel` instantiation is present, fits 256
threads in one CTA's registers, and takes no static shared memory, so its whole
request is the dynamic layout that `static_assert(kSmem <= 227 * 1024)` in
ffn_tf32.cu bounds to the 232,448 bytes a CTA may opt in to on sm_90."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "build", "csrc", "ffn_tf32.ptxas.log")
THREADS = 256
REGISTER_FILE = 65536
# (pad16(E), E's 40-float K-blocks): every instantiation fbbev_ffn_fwd launches
INSTANTIATIONS = {(16, 1), (32, 1), (48, 1), (48, 2), (64, 2), (80, 2)}


def _entries():
    if not os.path.exists(LOG):
        pytest.skip(f"ptxas log not built: {LOG}")
    entries, fn = {}, None
    for line in open(LOG):
        m = re.search(r"Compiling entry function '(\S*ffn_tf32_kernel\S*)'", line)
        if m:
            fn = m.group(1)
            continue
        m = re.search(r"Used (\d+) registers(.*)", line)
        if m and fn:
            smem = re.search(r"(\d+) bytes smem", m.group(2))
            entries[fn] = (int(m.group(1)), int(smem.group(1)) if smem else 0)
            fn = None
    return entries


def test_ffn_wgmma_not_serialised():
    """Any reason ptxas gives for serialising the MMAs (registers, C7511 /
    C7512; accumulator reads in flight, C7514; ...), not only C7515 / C7517."""
    _entries()
    bad = [line for line in open(LOG)
           if "ffn_tf32_kernel" in line and ("serialized" in line or "C7520" in line)]
    assert not bad, "".join(bad)


def test_ffn_instantiations_fit_one_cta():
    entries = _entries()
    found = set()
    for fn, (regs, smem) in entries.items():
        m = re.search(r"ffn_tf32_kernelILi(\d+)ELi(\d+)E", fn)
        assert m, fn
        found.add((int(m.group(1)), int(m.group(2))))
        assert regs * THREADS <= REGISTER_FILE, (fn, regs)
        assert smem == 0, (fn, smem)
    assert found == INSTANTIATIONS, found
