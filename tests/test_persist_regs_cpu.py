"""Register budget of the persistent forward loops (csrc/decoder_persist_tc.cu), read from ptxas at compile time.

lstm_loop_tc_kernel splits its registers between the roles with setmaxnreg: the MMA warpgroup gives up registers and the compute warps take
them.  ptxas silently falls back to the launch's uniform 168-register cap when it cannot honour a limit (it only says so in a -v remark),
and an inlined trap in the compute path has the same effect; either makes the attention loop spill heavily again (888 / 884 bytes of spill
stores / loads before the split).  No GPU is needed: ptxas reports the spills and the SASS shows the register limit instructions."""
import os
import re
import shutil
import subprocess

import pytest

from multilingual_text_to_speech_b200 import build

SRC = os.path.join(build.CSRC, 'decoder_persist_tc.cu')

# measured with the split in place: the attention loop (both memory-dim variants) keeps 44 / 44 bytes of spill stores / loads of
# loop-invariant values at its 224-register compute limit; the generator loop does not spill
SPILL_BOUND = {'<true,false>': 44, '<true,true>': 44, '<false,false>': 0}


def _nvcc():
    for cand in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', shutil.which('nvcc')):
        if cand and os.path.exists(cand):
            return cand
    return None


@pytest.fixture(scope='module')
def ptxas(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip('nvcc not available')
    out = tmp_path_factory.mktemp('regs')
    cubin = str(out / 'decoder_persist_tc.cubin')
    cmd = [nvcc] + build.NVCC_FLAGS + ['-I', os.path.join(build.ROOT, 'include'), '-Xptxas', '-v', '-cubin', SRC, '-o', cubin]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    cuobjdump = os.path.join(os.path.dirname(nvcc), 'cuobjdump')
    sass = subprocess.run([cuobjdump, '-sass', cubin], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout
    return res.stdout, sass


def _instantiation(mangled):
    m = re.search(r'lstm_loop_tc_kernelILb([01])ELb([01])E', mangled)
    return None if m is None else '<%s,%s>' % tuple('true' if b == '1' else 'false' for b in m.groups())


def _spills(log):
    """{instantiation: (spill store bytes, spill load bytes)} of the three lstm_loop_tc_kernel instantiations."""
    found = {}
    for m in re.finditer(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log):
        inst = _instantiation(m.group(1))
        if inst is not None:
            found[inst] = (int(m.group(3)), int(m.group(4)))
    return found


def test_register_split_is_honoured(ptxas):
    log, sass = ptxas
    assert "'setmaxnreg' ignored" not in log, 'ptxas dropped a setmaxnreg limit:\n' + log
    funcs = re.split(r'\n\s*Function : ', sass)[1:]
    loops = {_instantiation(f.split('\n')[0]): f for f in funcs if 'lstm_loop_tc_kernel' in f.split('\n')[0]}
    assert set(loops) == set(SPILL_BOUND), sorted(loops)
    for inst, body in loops.items():
        assert 'USETMAXREG.DEALLOC' in body and 'USETMAXREG.TRY_ALLOC' in body, f'{inst}: no register hand-over in the SASS'
    # the compute warps of the attention loop use more registers than the uniform 65536 / 384 = 168 cap would allow
    top = max(int(r) for r in re.findall(r'\bR(\d+)\b', loops['<true,false>']))
    assert top >= 168, top


def test_loops_stay_within_spill_bound(ptxas):
    found = _spills(ptxas[0])
    assert set(found) == set(SPILL_BOUND), found
    for inst, (stores, loads) in found.items():
        assert stores <= SPILL_BOUND[inst] and loads <= SPILL_BOUND[inst], f'{inst}: {stores} / {loads} bytes of spill stores / loads'
