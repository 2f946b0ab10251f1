"""CPU tier: accuracy of the branch-free log / sqrt / sin-cos of csrc/b2n_fastmath.cuh (used by the draws of the
lock-step rwalk kernels).  The header compiles for the host too; tests/fastmath_harness.cpp
compares it with long-double libm on the B2N uniforms (incl. arguments next to 0 and next to 1)."""
import json
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which('g++') is None, reason='no host compiler')
def test_fastmath_accuracy(tmp_path):
    exe = str(tmp_path / 'fm')
    subprocess.check_call(['g++', '-O2', '-ffp-contract=off', '-I', os.path.join(ROOT, 'dynesty_b200', 'csrc'), '-o', exe,
                           os.path.join(ROOT, 'tests', 'fastmath_harness.cpp'), '-lm'])
    r = json.loads(subprocess.check_output([exe, '1500000'], text=True))
    assert r['log_ulp'] <= 1.5 and r['rad_ulp'] <= 1.5 and r['sqrt_ulp'] <= 1.0 and r['div_ulp'] <= 1.0, r
    assert r['sin_ulp'] <= 2.5 and r['cos_ulp'] <= 2.5, r
