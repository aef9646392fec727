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
MODES = (0, 1, 2)          # kInfer, kTrainFwd, kBwd


def ffn_instantiations():
    """(NP2, KB1, MODE) of every ``ffn_tf32_kernel`` the three FFN entry points
    launch, by ffn_tf32.cu's ``dispatch`` rule over every width
    ``fbbev_ffn_supported`` takes: NP2 = pad16(E), KB1 = 2 (GEMM1 over two
    40-float K-blocks) when E > 40, else 1."""
    from fbbev_b200 import _lib
    L = _lib.lib()
    widths = [e for e in range(1, 129) if L.fbbev_ffn_supported(e, 80)]
    return {((e + 15) // 16 * 16, 2 if e > 40 else 1, mode)
            for e in widths for mode in MODES}


def ffn_kernel_args(name):
    """(NP2, KB1, MODE) of an ``ffn_tf32_kernel`` name, mangled or demangled;
    None for any other name."""
    m = (re.search(r"ffn_tf32_kernelILi(\d+)ELi(\d+)ELi(\d+)E", name) or
         re.search(r"ffn_tf32_kernel<\s*(\d+)\s*,\s*(\d+)\s*,\s*(\d+)\s*>", name))
    return tuple(int(v) for v in m.groups()) if m else None


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


def test_kernel_name_parser():
    assert ffn_kernel_args("_ZN5fbbev3ffn15ffn_tf32_kernelILi48ELi1ELi2EEEvNS0_9"
                           "ParamsForIXT1_EE4typeE") == (48, 1, 2)
    assert ffn_kernel_args("void fbbev::ffn::ffn_tf32_kernel<80, 2, 0>("
                           "fbbev::ffn::Params)") == (80, 2, 0)
    assert ffn_kernel_args("void fbbev::lnb::layernorm_bwd_kernel(float const*)") is None


def test_ffn_instantiations_fit_one_cta():
    """The kernels ptxas compiled == the dispatch rule's 18 (six (NP2, KB1)
    pairs in three modes): a new ``dispatch`` case fails here until the rule,
    and with it the GPU matrix's census, knows it."""
    entries = _entries()
    found = set()
    for fn, (regs, smem) in entries.items():
        args = ffn_kernel_args(fn)
        assert args, fn
        found.add(args)
        assert regs * THREADS <= REGISTER_FILE, (fn, regs)
        assert smem == 0, (fn, smem)
    want = ffn_instantiations()
    assert len(want) == 18
    assert found == want, (sorted(want - found), sorted(found - want))
