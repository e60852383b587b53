// Value windows for search by stored node and for the self-join through the C++ host mirror (gpu::EmbeddingIndex::SearchSimilar
// with windows, SearchPairs with a window and a band).
//   ./rows_pairs_windowed_mirror_test            (needs a GPU)      ./rows_pairs_windowed_mirror_test --no-gpu   (compiles and links only)
#include <cstdio>
#include <cstring>

#include "nornicdb_b200/host/nornic_cuda.hpp"

using namespace nornic;

int main(int argc, char **argv) {
    if (argc > 1 && std::strcmp(argv[1], "--no-gpu") == 0) {
        std::printf("rows and pairs windowed mirror ok\n");
        return 0;
    }
    int failures = 0;
    auto expect = [&](bool ok, const char *what) {
        if (!ok) { std::printf("FAIL: %s\n", what); ++failures; }
    };
    gpu::EmbeddingIndex ix(4);
    ix.Add("a", {1, 0, 0, 0});
    ix.Add("b", {0.9f, 0.1f, 0, 0});
    ix.Add("c", {0.8f, 0.2f, 0, 0});
    ix.Add("undated", {0.95f, 0.05f, 0, 0});
    // int64 timestamps t as keys t ^ 2^63 (nornicdb_b200.knn.value_keys); "undated" keeps key 0
    const uint64_t B = 1ull << 63;
    ix.SetRowValues(0, {B ^ 100, B ^ 200, B ^ 10000});
    auto all = ix.SearchSimilar({"a"}, 3);
    expect(all.size() == 1 && all[0].size() == 3 && all[0][0].ID == "undated", "no window: every other node");
    auto near = ix.SearchSimilar({"a", "missing", "c"}, 3, {}, {{B ^ 50, B ^ 250}, {0, ~0ull}, {B ^ 9000, B ^ 11000}});
    expect(near.size() == 3, "one list per id");
    expect(near[0].size() == 1 && near[0][0].ID == "b", "t in [50, 250]: the one other node inside, key 0 outside");
    expect(near[1].empty(), "a missing id: empty list");
    expect(near[2].empty(), "a window holding only the node itself: empty list");
    expect(ix.SearchPairs(0.5f).size() == 6, "no window, no band: every pair");
    auto band = ix.SearchPairs(0.5f, nullptr, nullptr, 150);
    expect(band.size() == 1 && band[0].A == "a" && band[0].B == "b", "band 150: the one pair of dated nodes close in time");
    const NkWindow late{B ^ 150, ~0ull};
    auto win = ix.SearchPairs(0.5f, nullptr, &late, NK_NO_GAP, 1);
    expect(win.size() == 1 && win[0].A == "b" && win[0].B == "c", "window t >= 150 on both sides, stripes of one row");
    std::printf(failures ? "%d FAILURES\n" : "rows and pairs windowed mirror ok\n", failures);
    return failures ? 1 : 0;
}
