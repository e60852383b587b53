// A filtered k-NN graph through the C++ host mirror (gpu::EmbeddingIndex::SimilarGraph(k, filters)): one "same collection"
// graph of a shared index, kept current across Remove, Add, SetRowTags (a node moving to another collection) and a changed
// filter: after each sequence the graph equals one built from scratch with the same tags and filters, and the index itself
// never rebuilt it.
//   ./graph_filtered_mirror_test            (needs a GPU)      ./graph_filtered_mirror_test --no-gpu   (compiles and links only)
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

// "same collection": the low 8 bits of a tag are its collection bit; bit 8 marks rows a few lists leave out
static std::vector<NkFilter> same_collection(const std::vector<uint64_t> &tags) {
    std::vector<NkFilter> f(tags.size());
    for (size_t r = 0; r < tags.size(); ++r) f[r] = NkFilter{0, r % 9 == 0 ? 1ull << 8 : 0ull, tags[r] & 0xffull};
    return f;
}

int main(int argc, char **argv) {
    if (argc > 1 && std::strcmp(argv[1], "--no-gpu") == 0) {
        std::printf("graph filtered mirror ok\n");
        return 0;
    }
    int failures = 0;
    auto expect = [&](bool ok, const std::string &what) {
        if (!ok) { std::printf("FAIL: %s\n", what.c_str()); ++failures; }
    };
    const int D = 64, K = 5;
    uint64_t state = 991;
    auto next = [&]() { state = state * 6364136223846793005ull + 1442695040888963407ull; return state >> 33; };
    auto vec = [&]() {
        std::vector<float> v(D);
        for (auto &x : v) x = (float)(next() % 2001) / 1000.0f - 1.0f;
        return v;
    };
    gpu::EmbeddingIndex ix(D);
    std::vector<std::vector<float>> seed;
    for (int i = 0; i < 400; ++i) { seed.push_back(vec()); ix.Add("n" + std::to_string(i), seed.back()); }
    // five collections of unequal size, the last one with 3 nodes (<= K: short lists)
    std::vector<uint64_t> tags(400);
    for (int i = 0; i < 400; ++i) {
        const int c = i < 200 ? 0 : i < 320 ? 1 : i < 380 ? 2 : i < 397 ? 3 : 4;
        tags[i] = (1ull << c) | ((next() & 1) << 8);
    }
    ix.SetRowTags(0, tags);
    auto g0 = ix.SimilarGraph(K, same_collection(ix.RowTags()));
    expect(g0.size() == 400 && ix.GraphRebuilds() == 1, "the first call builds the graph");
    expect(g0[399].size() == 2, "a three-node collection's list is short");
    auto check = [&](const std::string &what, std::vector<NkFilter> filters) {
        auto g = ix.SimilarGraph(K, filters);
        gpu::EmbeddingIndex fresh(D);
        fresh.Deserialize(ix.Serialize());
        fresh.SetRowTags(0, ix.RowTags());
        auto r = fresh.SimilarGraph(K, filters);
        expect(fresh.GraphRebuilds() == 1 && (int)g.size() == ix.Count() && same(g, r), what + " equals a rebuild");
        expect(ix.GraphRebuilds() == 1, what + ": no rebuild");
    };
    // Remove / Add into the small collection (a near copy of one of its nodes) and into the large one
    ix.Remove("n10");
    ix.Add("a0", seed[398]);
    ix.SetRowTags((uint64_t)ix.Count() - 1, {1ull << 4});
    ix.Add("a1", seed[399]);
    ix.SetRowTags((uint64_t)ix.Count() - 1, {1ull << 0});  // a copy of a small-collection node, in collection 0
    check("Remove / Add", same_collection(ix.RowTags()));
    // nodes move between collections; an Add rewrites a node in place
    ix.SetRowTags(17, {1ull << 2});
    ix.SetRowTags(250, {(1ull << 4) | (1ull << 8)});
    ix.Add("n33", vec());
    ix.Remove("n0");
    check("retag", same_collection(ix.RowTags()));
    // one node's filter widens to two collections, another's to none
    auto f = same_collection(ix.RowTags());
    f[5].any_of |= 1ull << 3;
    f[6] = NkFilter{0, 0, 0};
    check("filter change", f);
    for (int i = 0; i < 20; ++i) {
        ix.Remove("n" + std::to_string(40 + 7 * i));
        ix.Add("b" + std::to_string(i), vec());
        ix.SetRowTags((uint64_t)ix.Count() - 1, {1ull << (i % 5)});
    }
    f = same_collection(ix.RowTags());
    f[5].any_of |= 1ull << 3;
    f[6] = NkFilter{0, 0, 0};
    check("interleaved Add / Remove / retag", f);
    // SearchSimilar with one filter per id lists only admitted nodes
    auto s = ix.SearchSimilar({"n1", "n2"}, K, {NkFilter{0, 0, 1ull << 4}, NkFilter{~0ull, ~0ull, 0}});
    expect(s.size() == 2 && s[1].empty() && !s[0].empty() && s[0].size() <= (size_t)K, "SearchSimilar with filters");
    std::printf(failures ? "%d FAILURES\n" : "graph filtered mirror ok\n", failures);
    return failures ? 1 : 0;
}
