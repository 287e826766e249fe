"""The small tests of tests/test_gpu_pcisph.py against the host-emulated build of the same CUDA sources (tests/emu/),
once plain and once under AddressSanitizer, as tests/test_kernel_emulation.py does for the other solvers.  A check of
the kernel and host SOURCE, not of the sm_90a binary."""
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))

SMALL = "per_kernel_parity or overfull or steps_vs_oracle or device_side_loop"


def _run(lib, extra_env=None, at_least=4):
    env = dict(os.environ, SPH_EMU_LIB=lib, PYTHONPATH=ROOT)
    env.pop("SPH_B200_LIB", None)
    env.update(extra_env or {})
    cmd = [sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "-p", "no:cacheprovider", "-k", SMALL,
           os.path.join(ROOT, "tests", "test_gpu_pcisph.py")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, env=env, cwd=ROOT)
    tail = res.stdout[-3000:] + res.stderr[-3000:]
    assert res.returncode == 0, tail
    m = re.search(r"(\d+) passed", res.stdout)
    assert m and int(m.group(1)) >= at_least, tail
    assert "skipped" not in res.stdout.splitlines()[-1], tail


def test_pcisph_on_the_emulated_build():
    import build_emu
    _run(build_emu.build())


def test_pcisph_under_address_sanitizer():
    import build_emu
    asan_rt = subprocess.run(["/usr/bin/gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(asan_rt) or not os.path.exists(asan_rt):
        pytest.skip("libasan not available")
    _run(build_emu.build(asan=True), {"LD_PRELOAD": asan_rt, "ASAN_OPTIONS": "detect_leaks=0"})
