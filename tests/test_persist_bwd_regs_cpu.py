"""Register budget of the attention reverse loop (csrc/decoder_persist_bwd.cu), read from ptxas at compile time.

att_bwd_loop_kernel runs 256 threads at the 255-register maximum.  The cell backward's operands of the next step (gates, cell state,
d h static, keep masks), the recurrent partial sums and the query gradients reach shared memory by cp.async instead of through
registers; held in registers, the compiler parked them in local memory and the loop spilled 772 / 516 bytes (<96>) and 648 / 304
bytes (<80>) of spill stores / loads.  No GPU is needed: ptxas reports the spills."""
import os
import re
import shutil
import subprocess

import pytest

from multilingual_text_to_speech_b200 import build

SRC = os.path.join(build.CSRC, 'decoder_persist_bwd.cu')

# measured with the shared-memory staging and the out-of-line watchdog trap of mbar_wait: (spill store bytes, spill load bytes) of each
# instantiation
SPILL_BOUND = {'<96>': (204, 136), '<80>': (72, 48)}


def _nvcc():
    for cand in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', shutil.which('nvcc')):
        if cand and os.path.exists(cand):
            return cand
    return None


@pytest.fixture(scope='module')
def ptxas_log(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip('nvcc not available')
    out = tmp_path_factory.mktemp('bwd_regs')
    cmd = [nvcc] + build.NVCC_FLAGS + ['-I', os.path.join(build.ROOT, 'include'), '-Xptxas', '-v', '-cubin', SRC,
                                       '-o', str(out / 'decoder_persist_bwd.cubin')]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    return res.stdout


def test_attention_reverse_loop_stays_within_spill_bound(ptxas_log):
    found = {}
    for m in re.finditer(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
                         ptxas_log):
        inst = re.search(r'att_bwd_loop_kernelILi(\d+)EE', m.group(1))
        if inst is not None:
            found['<%s>' % inst.group(1)] = (int(m.group(3)), int(m.group(4)))
    assert set(found) == set(SPILL_BOUND), found
    for inst, (stores, loads) in found.items():
        bound_st, bound_ld = SPILL_BOUND[inst]
        assert stores <= bound_st and loads <= bound_ld, f'{inst}: {stores} / {loads} bytes of spill stores / loads'
