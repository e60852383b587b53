// The k-NN graph through the C++ host mirror (gpu::EmbeddingIndex::SimilarGraph), kept current across Remove as well as
// Add / AddBatch: after each sequence the graph equals one built from scratch, and the index itself never rebuilt it.
//   ./graph_remove_mirror_test            (needs a GPU)      ./graph_remove_mirror_test --no-gpu   (compiles and links only)
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
        std::printf("graph remove mirror ok\n");
        return 0;
    }
    int failures = 0;
    auto expect = [&](bool ok, const std::string &what) {
        if (!ok) { std::printf("FAIL: %s\n", what.c_str()); ++failures; }
    };
    const int D = 64, K = 5;
    uint64_t state = 777;
    auto vec = [&]() {
        std::vector<float> v(D);
        for (auto &x : v) { state = state * 6364136223846793005ull + 1442695040888963407ull; x = (float)((state >> 40) % 2001) / 1000.0f - 1.0f; }
        return v;
    };
    gpu::EmbeddingIndex ix(D);
    // the same nodes in the same rows (Serialize keeps the row order), their graph built from scratch
    auto check = [&](const std::string &what) {
        auto g = ix.SimilarGraph(K);
        gpu::EmbeddingIndex fresh(D);
        fresh.Deserialize(ix.Serialize());
        auto r = fresh.SimilarGraph(K);
        expect(fresh.GraphRebuilds() == 1 && (int)g.size() == ix.Count() && same(g, r), what + " equals a rebuild");
        expect(ix.GraphRebuilds() == 1, what + ": no rebuild");
    };
    for (int i = 0; i < 400; ++i) ix.Add("n" + std::to_string(i), vec());
    auto g0 = ix.SimilarGraph(K);
    expect(g0.size() == 400 && ix.GraphRebuilds() == 1, "the first call builds the graph");
    // Remove only: a middle row, the last row, the first row
    ix.Remove("n200");  // n399 moves into row 200
    ix.Remove("n398");  // the last row now
    ix.Remove("n0");    // n397 moves into row 0
    check("Remove");
    // Add / Remove / Add: an appended node removed again, a moved node rewritten, an append after a removal
    ix.AddBatch({"a0", "a1", "a2"}, {vec(), vec(), vec()});
    ix.Remove("a1");
    ix.Add("n5", vec());
    ix.Add("n397", vec());
    ix.Remove("n17");
    ix.Add("a3", vec());
    check("Add / Remove / Add");
    for (int i = 0; i < 30; ++i) {
        ix.Remove("n" + std::to_string(30 + 3 * i));
        ix.Add("b" + std::to_string(i), vec());
    }
    check("interleaved Add / Remove");
    ix.Remove("b29");  // the last row: nothing moves
    check("Remove of the last row");
    std::printf(failures ? "%d FAILURES\n" : "graph remove mirror ok\n", failures);
    return failures ? 1 : 0;
}
