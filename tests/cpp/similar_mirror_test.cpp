// Search by stored node through the C++ host mirror (gpu::EmbeddingIndex::SearchSimilar).
//   ./similar_mirror_test            (needs a GPU)      ./similar_mirror_test --no-gpu   (compiles and links only)
#include <cstdio>
#include <cstring>

#include "nornicdb_b200/host/nornic_cuda.hpp"

using namespace nornic;

int main(int argc, char **argv) {
    if (argc > 1 && std::strcmp(argv[1], "--no-gpu") == 0) {
        std::printf("similar mirror ok\n");
        return 0;
    }
    int failures = 0;
    auto expect = [&](bool ok, const char *what) {
        if (!ok) { std::printf("FAIL: %s\n", what); ++failures; }
    };
    gpu::EmbeddingIndex ix(4);
    expect(ix.SearchSimilar({"a"}, 3)[0].empty(), "empty index: an empty list");
    ix.Add("a", {1, 0, 0, 0});
    ix.Add("b", {0.9f, 0.1f, 0, 0});
    ix.Add("c", {0, 1, 0, 0});
    ix.Add("d", {1, 0, 0, 0});
    auto r = ix.SearchSimilar({"a", "missing", "c", "a"}, 2);
    expect(r.size() == 4, "one list per id");
    expect(r[0].size() == 2 && r[0][0].ID == "d" && r[0][1].ID == "b", "a: its duplicate d first, never itself");
    expect(r[1].empty(), "a missing id gets an empty list");
    expect(r[2].size() == 2 && r[2][0].ID == "b" && r[2][1].ID == "a", "c: b, then a (tie with d, lower row)");
    expect(r[3].size() == 2 && r[3][0].ID == "d", "repeated id, same answer");
    auto all = ix.SearchSimilar({"b"}, 10);
    expect(all[0].size() == 3 && all[0][0].ID == "a" && all[0][1].ID == "d" && all[0][2].ID == "c", "k above the other nodes: all of them");
    ix.Remove("a");  // d moves into a's row
    auto moved = ix.SearchSimilar({"d", "a"}, 1);
    expect(moved[0].size() == 1 && moved[0][0].ID == "b" && moved[1].empty(), "after swap-remove");
    std::printf(failures ? "%d FAILURES\n" : "similar mirror ok\n", failures);
    return failures ? 1 : 0;
}
