// host_mirror_test.cpp — the reference's own GPU-boundary tests (pkg/gpu/cuda/cuda_test.go, pkg/gpu/gpu_test.go),
// replayed against the C++ host mirror (nornicdb_b200/host/nornic_cuda.hpp) over libnornic_knn.so.
//   g++ -std=c++17 -I. tests/cpp/host_mirror_test.cpp -Lnornicdb_b200 -lnornic_knn -Wl,-rpath,$PWD/nornicdb_b200 -o host_mirror_test
//   ./host_mirror_test            (needs a GPU)      ./host_mirror_test --no-gpu   (error paths only)
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "nornicdb_b200/host/nornic_cuda.hpp"

using namespace nornic;
static int failures = 0;
#define CHECK(cond) do { if (!(cond)) { std::printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #cond); ++failures; } } while (0)
static bool near(float a, float b, float tol = 1e-3f) { return std::fabs(a - b) <= tol; }

static void test_no_gpu() {
    CHECK(!cuda::IsAvailable());
    CHECK(cuda::DeviceCount() == 0);
    bool threw = false;
    try { cuda::NewDevice(0); } catch (const cuda::ErrCUDANotAvailable &) { threw = true; }
    CHECK(threw);  // cuda_bridge.go:446-448
    threw = false;
    try { gpu::EmbeddingIndex ei(4); } catch (const cuda::CudaError &) { threw = true; }
    CHECK(threw);  // no CPU fallback: the index cannot exist without a device
}

static void test_cuda_package() {
    auto device = cuda::NewDevice(0);
    CHECK(device->ID() == 0 && !device->Name().empty() && device->MemoryMB() > 0);
    CHECK(device->ComputeCapability().first == 9);
    {   // cuda_test.go:215-253 TestNormalizeVectors
        auto buf = device->NewBuffer({3, 4, 0, 1, 0, 0});
        device->NormalizeVectors(*buf, 2, 3);
        auto r = buf->ReadFloat32(6);
        CHECK(near(r[0], 0.6f) && near(r[1], 0.8f) && near(r[2], 0) && near(r[3], 1) && near(r[4], 0) && near(r[5], 0));
    }
    {   // cuda_test.go:255-312 TestCosineSimilarity
        auto emb = device->NewBuffer({1, 0, 0, 0, 1, 0, 0.6f, 0.8f, 0});
        auto q = device->NewBuffer({1, 0, 0});
        auto sc = device->NewEmptyBuffer(3);
        device->CosineSimilarity(*emb, *q, *sc, 3, 3, true);
        auto s = sc->ReadFloat32(3);
        CHECK(near(s[0], 1.0f) && near(s[1], 0.0f) && near(s[2], 0.6f));
    }
    {   // cuda_test.go:314-353 TestTopK
        auto sc = device->NewBuffer({0.1f, 0.8f, 0.3f, 0.9f, 0.2f});
        auto r = device->TopK(*sc, 5, 3);
        CHECK(r.first.size() == 3 && r.first[0] == 3 && r.first[1] == 1 && r.first[2] == 2);
    }
    {   // cuda_test.go:355-400 TestSearch
        auto emb = device->NewBuffer({1, 0, 0, 0, 1, 0, 0, 0, 1, 0.6f, 0.8f, 0, 0.7f, 0.7f, 0.14f});
        auto res = device->Search(*emb, {0.6f, 0.8f, 0.0f}, 5, 3, 2, true);
        CHECK(res.size() == 2 && res[0].Index == 3 && near(res[0].Score, 1.0f));
        CHECK(device->Search(*emb, {0.6f, 0.8f, 0.0f}, 5, 3, 0, true).empty());   // cuda_test.go:402-431 k=0 -> nil
        CHECK(device->Search(*emb, {1, 0, 0}, 5, 3, 10, true).size() == 5);        // cuda_test.go:433-462 k>n -> n
        auto batch = device->SearchBatch(*emb, {0.6f, 0.8f, 0, 0, 0, 1}, 2, 5, 3, 1, cuda::Metric::Cosine);
        CHECK(batch.size() == 2 && batch[0][0].Index == 3 && batch[1][0].Index == 2);
    }
    {   // buffers: cuda_bridge.go:507-509, 574-576
        bool threw = false;
        try { device->NewBuffer({}); } catch (const cuda::CudaError &) { threw = true; }
        CHECK(threw);
        auto b = device->NewBuffer({1, 2, 3}, cuda::MemoryPinned);
        CHECK(b->Size() == 12 && b->ReadFloat32(4).empty() && b->ReadFloat32(2).size() == 2);
        b->Release();
        b->Release();
    }
}

static void test_embedding_index() {
    {   // gpu_test.go:496-533 TestEmbeddingIndexAddAndSearch
        gpu::EmbeddingIndex ei(4);
        ei.Add("node-1", {1, 0, 0, 0});
        ei.Add("node-2", {0, 1, 0, 0});
        ei.Add("node-3", {0.9f, 0.1f, 0, 0});
        ei.Add("node-4", {0, 0, 1, 0});
        CHECK(ei.Count() == 4);
        auto r = ei.Search({1, 0, 0, 0}, 2);
        CHECK(r.size() == 2 && r[0].ID == "node-1" && r[0].Score >= 0.99f && r[1].ID == "node-3");
        bool threw = false;
        try { ei.Search({1, 0, 0}, 1); } catch (const gpu::ErrInvalidDimensions &) { threw = true; }
        CHECK(threw);  // gpu.go:1533-1535
        // Remove = swap with last (gpu.go:1437-1471); ids still map to the right rows
        CHECK(ei.Remove("node-1") && !ei.Remove("node-1") && ei.Count() == 3 && !ei.Has("node-1"));
        r = ei.Search({1, 0, 0, 0}, 1);
        CHECK(r.size() == 1 && r[0].ID == "node-3");
        r = ei.Search({0, 0, 1, 0}, 1);
        CHECK(r[0].ID == "node-4" && r[0].Score >= 0.99f);
        // update in place (gpu.go:1391-1399)
        ei.Add("node-2", {0, 0, 2, 0});
        r = ei.Search({0, 0, 1, 0}, 2);
        CHECK(r.size() == 2 && ((r[0].ID == "node-4" && r[1].ID == "node-2") || (r[0].ID == "node-2" && r[1].ID == "node-4")));
    }
    {   // gpu_test.go:1592-1621 TestEmbeddingIndexScoreSubsetCPU (here: on the device)
        gpu::EmbeddingIndex ei(3);
        ei.Add("a", {1, 0, 0});
        ei.Add("b", {0, 1, 0});
        ei.Add("c", {1, 1, 0});
        auto r = ei.ScoreSubset({1, 0, 0}, {"b", "c", "a", "missing"});
        CHECK(r.size() == 3 && r[0].ID == "a" && r[1].ID == "c" && r[2].ID == "b");
        CHECK(ei.ScoreSubset({1, 0, 0}, {}).empty());
        // Serialize / Deserialize round trip (gpu.go:2373-2454)
        auto blob = ei.Serialize();
        CHECK(blob.size() == 8 + 3 * 5 + 9 * 4 && blob[0] == 3 && blob[4] == 3);
        gpu::EmbeddingIndex other(3);
        other.Deserialize(blob);
        auto r2 = other.Search({1, 0, 0}, 3);
        CHECK(r2.size() == 3 && r2[0].ID == "a" && r2[1].ID == "c" && r2[2].ID == "b");
        std::vector<float> v;
        CHECK(other.Get("c", &v) && v.size() == 3 && v[0] == 1 && v[1] == 1 && v[2] == 0);
        bool threw = false;
        try { gpu::EmbeddingIndex wrong(5); wrong.Deserialize(blob); } catch (const gpu::ErrInvalidDimensions &) { threw = true; }
        CHECK(threw);
    }
}

int main(int argc, char **argv) {
    const bool no_gpu = argc > 1 && std::strcmp(argv[1], "--no-gpu") == 0;
    if (no_gpu) test_no_gpu();
    else {
        if (!cuda::IsAvailable()) { std::printf("FAIL: no CUDA device (use --no-gpu for the error-path checks)\n"); return 2; }
        test_cuda_package();
        test_embedding_index();
    }
    std::printf(failures ? "%d FAILURES\n" : "host mirror ok\n", failures);
    return failures ? 1 : 0;
}
