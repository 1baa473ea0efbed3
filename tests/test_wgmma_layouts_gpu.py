"""Known-answer check of the wgmma operand layouts (K-major and transposed chunk-major images, descriptor strides and
K advances) for every N the field and WGRAD kernels use: exact integer products, so a layout error cannot hide inside
the end-to-end parity tolerances.  The program is built by __graft_entry__.build() (tests/cuda/Makefile)."""
import os
import subprocess

import pytest

PROBE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cuda", "wgmma_layout_probe")


@pytest.mark.gpu
def test_wgmma_operand_layouts_known_answer():
    assert os.path.exists(PROBE), "tests/cuda/wgmma_layout_probe is missing: run __graft_entry__.build()"
    r = subprocess.run([PROBE], capture_output=True, text=True, timeout=120)
    print(r.stdout)
    assert r.returncode == 0 and "all ok" in r.stdout, r.stdout + r.stderr
