"""Generates tests/golden/dropin_golden.pt: the 'reference' arm of tests/test_reference_code_dropin.py (the reference's
own saver / loader / evaluate code driving this engine) for 1 and 2 stages, plus the resume leg.

Run in the build container only (needs /root/reference):   python tests/golden/make_golden_dropin.py
"""
import os
import sys
import tempfile

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
OUT = os.path.join(HERE, 'dropin_golden.pt')


def main():
    sys.path.insert(0, TESTS)
    import test_reference_code_dropin as T
    out = {}
    for world in (1, 2):
        with tempfile.TemporaryDirectory() as d:
            out[str(world)] = T.run_record(world, 'reference', d)
    torch.save(out, OUT)
    print(OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()
