"""gs::BinList's rules (csrc/gs_internal.cuh), compiled with the library's nvcc flags against a model of the list in place of
its buffers and CUDA calls, and run without a device: the capacity clamp, growth to the total plus a quarter (capped at
768 Mi, none above it), which draws read the list back, and the overflow flag across the draws of a public call."""
import subprocess
from pathlib import Path

from unitygaussiansplatting_b200 import build

ROOT = Path(__file__).resolve().parents[1]


def test_bin_list_rules(tmp_path):
    exe = tmp_path / "bin_list_test"
    subprocess.run([build._nvcc(), *build.nvcc_flags(), "-I", str(build.CSRC), "-o", str(exe), str(ROOT / "tests" / "bin_list_test.cu")],
                   check=True, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    r = subprocess.run([str(exe)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
