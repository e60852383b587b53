"""The C++ host mirror's windowed k-NN graph (gpu::EmbeddingIndex::SimilarGraph(k, filters, windows)) compiles against the C
ABI, and keeps a time-local graph of a small index current across SetRowValues, Remove, Add and a window change on the GPU
without rebuilding it."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def graph_windowed_binary(knn_lib, tmp_path_factory):
    src = os.path.join(ROOT, "tests", "cpp", "graph_windowed_mirror_test.cpp")
    lib = os.path.join(ROOT, "nornicdb_b200", "libnornic_knn.so")
    out = str(tmp_path_factory.mktemp("cpp") / "graph_windowed_mirror_test")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-I", ROOT, src, "-L", os.path.dirname(lib), "-lnornic_knn",
                    f"-Wl,-rpath,{os.path.dirname(lib)}", "-lpthread", "-o", out], check=True, cwd=ROOT)
    return out


def test_graph_windowed_mirror_compiles(graph_windowed_binary):
    out = subprocess.run([graph_windowed_binary, "--no-gpu"], capture_output=True, text=True)
    assert out.returncode == 0 and "graph windowed mirror ok" in out.stdout


@pytest.mark.gpu
def test_graph_windowed_mirror_on_gpu(graph_windowed_binary):
    out = subprocess.run([graph_windowed_binary], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "graph windowed mirror ok" in out.stdout
