"""Known-answer check of the register-A (RS) wgmma at N = 64, which DGRAD runs its embedding steps (L5e^T, L0^T) in, and
of the skip layer's pattern: one set of A fragments feeds an N = 64 MMA and then, unchanged, an N = 256 MMA.  Both must be
bit-identical to the shared-memory MMA on the same fp16 image and to the exact integer product.  The program is built
by __graft_entry__.build() (tests/cuda/wgmma_rs64_probe.mk)."""
import os
import subprocess

import pytest

PROBE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cuda", "wgmma_rs64_probe")


@pytest.mark.gpu
def test_wgmma_register_a_n64_and_shared_fragments_known_answer():
    assert os.path.exists(PROBE), "tests/cuda/wgmma_rs64_probe is missing: run __graft_entry__.build()"
    r = subprocess.run([PROBE], capture_output=True, text=True, timeout=120)
    print(r.stdout)
    assert r.returncode == 0 and "all ok" in r.stdout, r.stdout + r.stderr
