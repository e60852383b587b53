"""The C++ host mirror's self-join kept current (gpu::EmbeddingIndex::SimilarPairs and PairsOfNodes) compiles against the C ABI,
and on the GPU keeps the join of a small index equal to a fresh index's across Add, AddBatch, Remove, SetRowTags and
SetRowValues without rebuilding it."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def pairs_update_binary(knn_lib, tmp_path_factory):
    src = os.path.join(ROOT, "tests", "cpp", "pairs_update_mirror_test.cpp")
    lib = os.path.join(ROOT, "nornicdb_b200", "libnornic_knn.so")
    out = str(tmp_path_factory.mktemp("cpp") / "pairs_update_mirror_test")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-I", ROOT, src, "-L", os.path.dirname(lib), "-lnornic_knn",
                    f"-Wl,-rpath,{os.path.dirname(lib)}", "-lpthread", "-o", out], check=True, cwd=ROOT)
    return out


def test_pairs_update_mirror_compiles(pairs_update_binary):
    out = subprocess.run([pairs_update_binary, "--no-gpu"], capture_output=True, text=True)
    assert out.returncode == 0 and "pairs update mirror ok" in out.stdout


@pytest.mark.gpu
def test_pairs_update_mirror_on_gpu(pairs_update_binary):
    out = subprocess.run([pairs_update_binary], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "pairs update mirror ok" in out.stdout
