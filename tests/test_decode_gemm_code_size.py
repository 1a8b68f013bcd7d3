"""CPU: the machine code of every production decode-GEMM kernel (gemm_tc_kernel, one per epilogue kind x tile width x passes) stays under a
ceiling.  An epilogue that inlines every option walked 70-170 KB of straight-line code per tile, more than an SM's instruction cache
holds, and every CTA fetched it from L2 at the same moment (DESIGN §6.1).  The ceiling keeps the epilogue from growing back one option at
a time.  Reads the built library with cuobjdump; skips when either is missing."""
import os
import re
import shutil
import subprocess

import pytest

from helpers import REPO

LIB = os.path.join(REPO, 'imagecaptioning.pytorch_b200', 'libcapb200.so')
CEILING_KB = 64
KERNEL = re.compile(r'gemm_tc_kernelILi(\d+)ELi(\d+)ELi(\d+)ELb([01])E')


def _cuobjdump():
    for cand in (shutil.which('cuobjdump'), '/usr/local/cuda/bin/cuobjdump'):
        if cand and os.path.exists(cand):
            return cand
    return None


def test_decode_gemm_kernels_fit_the_ceiling():
    tool = _cuobjdump()
    if tool is None or not os.path.exists(LIB):
        pytest.skip('needs cuobjdump and the built library')
    sass = subprocess.run([tool, '-sass', LIB], capture_output=True, text=True, check=True).stdout
    sizes = {}
    for chunk in re.split(r'\n\s*Function : ', sass)[1:]:
        m = KERNEL.search(chunk.split('\n', 1)[0])
        if m is None or m.group(4) == '1':           # TRACE = true: the diagnostic build of tools/gemm_trace.py
            continue
        n_instr = len(re.findall(r'/\*[0-9a-f]{4,}\*/\s+[^;\n]*;', chunk))
        sizes['BN %s, %s-pass, kind %s' % m.groups()[:3]] = n_instr * 16           # sm_90 instructions are 16 bytes
    assert len(sizes) == 3 * 3 * 2, sorted(sizes)     # kind x BN x passes
    over = {k: v for k, v in sizes.items() if v > CEILING_KB * 1024}
    assert not over, over
