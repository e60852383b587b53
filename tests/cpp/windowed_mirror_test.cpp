// Per-query value windows through the C++ host mirror (gpu::EmbeddingIndex::SetRowValues / SearchBatchWindowed / SearchRange).
//   ./windowed_mirror_test            (needs a GPU)      ./windowed_mirror_test --no-gpu   (compiles and links only)
#include <cstdio>
#include <cstring>

#include "nornicdb_b200/host/nornic_cuda.hpp"

using namespace nornic;

int main(int argc, char **argv) {
    if (argc > 1 && std::strcmp(argv[1], "--no-gpu") == 0) {
        std::printf("windowed mirror ok\n");
        return 0;
    }
    int failures = 0;
    auto expect = [&](bool ok, const char *what) {
        if (!ok) { std::printf("FAIL: %s\n", what); ++failures; }
    };
    gpu::EmbeddingIndex ix(4);
    ix.Add("old-a", {1, 0, 0, 0});
    ix.Add("new-b", {0.9f, 0.1f, 0, 0});
    ix.Add("new-c", {0, 1, 0, 0});
    ix.Add("undated", {0.95f, 0.05f, 0, 0});
    // int64 timestamps t as keys t ^ 2^63 (nornicdb_b200.knn.value_keys); "undated" keeps key 0
    const uint64_t B = 1ull << 63;
    ix.SetRowValues(0, {B ^ 100, B ^ 200, B ^ 300});
    const std::vector<float> q = {1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0};
    const std::vector<NkWindow> w = {{0, ~0ull}, {B ^ 150, ~0ull}, {B ^ 400, ~0ull}};
    auto r = ix.SearchBatchWindowed(q, {}, w, 3, 4);
    expect(r.size() == 3, "one result list per query");
    expect(r[0].size() == 4 && r[0][0].ID == "old-a" && r[0][1].ID == "undated", "{0, ~0}: every row");
    expect(r[1].size() == 2 && r[1][0].ID == "new-b" && r[1][1].ID == "new-c", "t >= 150: only the newer rows, the rest padding");
    expect(r[2].empty(), "a window past every value: no row");
    const std::vector<NkFilter> f = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    auto g = ix.SearchRange(q, {0.5f, 0.5f, 0.5f}, f, {{0, ~0ull}, {B ^ 150, B ^ 250}, {1, ~0ull}}, 3);
    expect(g[0].size() == 3, "range, no window: every row above the threshold");
    expect(g[1].size() == 1 && g[1][0].ID == "new-b", "range, closed window: the one row inside");
    expect(g[2].size() == 2 && g[2][0].ID == "old-a" && g[2][1].ID == "new-b", "range, lo = 1: rows without a value never match");
    std::printf(failures ? "%d FAILURES\n" : "windowed mirror ok\n", failures);
    return failures ? 1 : 0;
}
