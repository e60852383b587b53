"""The C++ host mirror's windowed search by stored node and windowed self-join (gpu::EmbeddingIndex::SearchSimilar with windows,
SearchPairs with a window and a band) compile against the C ABI, and answer a tiny dated index on the GPU."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def mirror_binary(knn_lib, tmp_path_factory):
    src = os.path.join(ROOT, "tests", "cpp", "rows_pairs_windowed_mirror_test.cpp")
    lib = os.path.join(ROOT, "nornicdb_b200", "libnornic_knn.so")
    out = str(tmp_path_factory.mktemp("cpp") / "rows_pairs_windowed_mirror_test")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-I", ROOT, src, "-L", os.path.dirname(lib), "-lnornic_knn",
                    f"-Wl,-rpath,{os.path.dirname(lib)}", "-lpthread", "-o", out], check=True, cwd=ROOT)
    return out


def test_rows_pairs_windowed_mirror_compiles(mirror_binary):
    out = subprocess.run([mirror_binary, "--no-gpu"], capture_output=True, text=True)
    assert out.returncode == 0 and "rows and pairs windowed mirror ok" in out.stdout


@pytest.mark.gpu
def test_rows_pairs_windowed_mirror_on_gpu(mirror_binary):
    out = subprocess.run([mirror_binary], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "rows and pairs windowed mirror ok" in out.stdout
