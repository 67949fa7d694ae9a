"""Every selectable round ordering (DM_KERNEL_VARIANT) is bit-exact on the GPU, not only the default.

Each runs in a process of its own (the variant is read once, at engine creation).  The default deep variant
(8: round form 7, two warps per stream in launches of at most 264 jobs) is what tests/test_gpu_parity.py exercises on every kernel shape; here the alternatives that stay
selectable for A/B runs - ptxas' own ordering (0), the other short-chain forms (4, 5) and the wide kernel with
cp.async-staged lines (21) - are held to the
same bar by tools/check_variant.py: every length 0..300, group / line boundaries, 1500 ragged blobs in one
launch, the fused CAS copy, on the deep, 2/4/8/16-streams-per-warp and wide kernels, against hashlib.
The arithmetic of every round form is also proven on the host by tests/test_native_host.py.
"""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["9,0", "9,4", "9,5", "21,7"])   # wide 9 / 21 x deep 0, 4, 5, 7
def test_alternative_round_orderings_are_bit_exact_on_the_gpu(variant):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "check_variant.py"), variant],
                         capture_output=True, text=True, timeout=240)
    print(out.stdout[-3000:])
    assert out.returncode == 0 and "VARIANT OK" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]
