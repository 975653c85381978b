"""Golden vectors of the module-level cases (tests/module_cases.py) from the UNMODIFIED reference's classes (CPU, fp32).

    python tests/golden/make_golden_modules.py        # needs the reference checkout at REF; writes tests/golden/modules.npz

The reference is imported read-only; only its module classes run.  tests/test_gpu_modules.py compares this package's classes on the
GPU against the stored results.
"""
import os
import sys

import numpy as np

REF = '/root/reference'
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))


def main():
    sys.path.insert(0, REF)
    sys.dont_write_bytecode = True
    import torch
    import utils  # noqa: F401  (must precede the modules: circular import in the reference)
    from modules.layers import ZoneoutLSTMCell, DropoutLSTMCell
    from modules.generated import Conv1dGenerated, BatchNorm1dGenerated
    from modules.attention import LocationSensitiveAttention
    import module_cases as C

    torch.manual_seed(0)
    out = {}
    I, H = 544, 1024
    out.update(C.pack('lstm_zoneout', C.lstm_case('zoneout', ZoneoutLSTMCell(I, H, 0.1, 0.1), 'cpu')))
    out.update(C.pack('lstm_dropout', C.lstm_case('dropout', DropoutLSTMCell(I, H, 0.1), 'cpu')))
    G, gd, bn, Cin, Cout, k, dil = 3, 6, 4, 8, 12, 3, 2
    for train in (True, False):
        conv = Conv1dGenerated(gd, bn, G * Cin, G * Cout, k, padding=0, dilation=dil, groups=G, bias=False)
        norm = BatchNorm1dGenerated(gd, bn, G * Cout, groups=G)
        out.update(C.pack(f'conv_train{int(train)}', C.conv_case(train, conv, norm, 'cpu')))
    d = C.ATT_DIMS
    out.update(C.pack('attention', C.attention_case(LocationSensitiveAttention(d['K'], d['C'], False, d['A'], d['D'], d['M']), 'cpu')))
    path = os.path.join(HERE, 'modules.npz')
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), 'bytes,', len(out), 'arrays')


if __name__ == '__main__':
    main()
