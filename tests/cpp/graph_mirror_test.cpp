// The k-NN graph through the C++ host mirror (gpu::EmbeddingIndex::SimilarGraph), kept current across Add / AddBatch.
//   ./graph_mirror_test            (needs a GPU)      ./graph_mirror_test --no-gpu   (compiles and links only)
#include <cstdio>
#include <cstring>
#include <string>

#include "nornicdb_b200/host/nornic_cuda.hpp"

using namespace nornic;

static bool same(const std::vector<std::vector<gpu::SearchResult>> &a, const std::vector<std::vector<gpu::SearchResult>> &b) {
    if (a.size() != b.size()) return false;
    for (size_t i = 0; i < a.size(); ++i) {
        if (a[i].size() != b[i].size()) return false;
        for (size_t j = 0; j < a[i].size(); ++j)
            if (a[i][j].ID != b[i][j].ID || std::memcmp(&a[i][j].Score, &b[i][j].Score, 4) != 0) return false;
    }
    return true;
}

int main(int argc, char **argv) {
    if (argc > 1 && std::strcmp(argv[1], "--no-gpu") == 0) {
        std::printf("graph mirror ok\n");
        return 0;
    }
    int failures = 0;
    auto expect = [&](bool ok, const char *what) {
        if (!ok) { std::printf("FAIL: %s\n", what); ++failures; }
    };
    const int D = 64, K = 5;
    uint64_t state = 12345;
    auto vec = [&]() {
        std::vector<float> v(D);
        for (auto &x : v) { state = state * 6364136223846793005ull + 1442695040888963407ull; x = (float)((state >> 40) % 2001) / 1000.0f - 1.0f; }
        return v;
    };
    gpu::EmbeddingIndex ix(D), ref(D);
    auto add = [&](const std::string &id, const std::vector<float> &v) { ix.Add(id, v); ref.Add(id, v); };
    for (int i = 0; i < 400; ++i) add("n" + std::to_string(i), vec());
    auto g0 = ix.SimilarGraph(K);
    expect(g0.size() == 400 && g0[0].size() == (size_t)K, "one list of k per node");
    for (int i = 400; i < 460; ++i) add("n" + std::to_string(i), vec());  // appended
    add("n7", vec());                                                    // rewritten
    add("n7", vec());                                                    // and again
    auto g1 = ix.SimilarGraph(K);   // updated
    auto r1 = ref.SimilarGraph(K);  // the reference index builds its graph from scratch
    expect(same(g1, r1), "updated graph equals a rebuild after Add / AddBatch");
    ix.Remove("n3");
    ref.Remove("n3");
    auto g2 = ix.SimilarGraph(K);   // rebuilt after Remove
    expect(g2.size() == 459 && same(g2, ref.SimilarGraph(K)), "rebuilt after Remove");
    std::printf(failures ? "%d FAILURES\n" : "graph mirror ok\n", failures);
    return failures ? 1 : 0;
}
