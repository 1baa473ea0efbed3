"""Known-answer check of the register-A (RS) wgmma form and of the accumulator -> A-fragment packing (frag_pair) that
the forward kernel chains its trunk layers with: bit-identical to the shared-memory MMA on the same fp16 image and to
the exact integer product, for every N used in RS form.  The program is built by __graft_entry__.build()
(tests/cuda/wgmma_rs_probe.mk)."""
import os
import subprocess

import pytest

PROBE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cuda", "wgmma_rs_probe")


@pytest.mark.gpu
def test_wgmma_register_a_known_answer():
    assert os.path.exists(PROBE), "tests/cuda/wgmma_rs_probe is missing: run __graft_entry__.build()"
    r = subprocess.run([PROBE], capture_output=True, text=True, timeout=120)
    print(r.stdout)
    assert r.returncode == 0 and "all ok" in r.stdout, r.stdout + r.stderr
