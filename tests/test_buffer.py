"""gs::Buffer (csrc/gs_buffer.cuh), the owner of every scratch buffer the library grows, compiled on its own with the
library's nvcc flags: a reserve that fails leaves the buffer empty, so a later smaller reserve allocates instead of
returning a null pointer behind a stale size."""
import subprocess
from pathlib import Path

import pytest

from conftest import has_cuda
from unitygaussiansplatting_b200 import build

ROOT = Path(__file__).resolve().parents[1]


def _run(tmp_path, mode):
    exe = tmp_path / "buffer_test"
    subprocess.run([build._nvcc(), *build.nvcc_flags(), "-I", str(build.CSRC), "-o", str(exe), str(ROOT / "tests" / "buffer_test.cu")],
                   check=True, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    return subprocess.run([str(exe), mode], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)


@pytest.mark.skipif(has_cuda(), reason="CPU-only behaviour")
def test_reserve_without_a_device_leaves_the_buffer_empty(tmp_path):
    r = _run(tmp_path, "no-device")
    assert r.returncode == 0, r.stdout


@pytest.mark.gpu
@pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")
def test_reserve_grows_keeps_fails_empty_and_recovers(tmp_path):
    r = _run(tmp_path, "device")
    assert r.returncode == 0, r.stdout
