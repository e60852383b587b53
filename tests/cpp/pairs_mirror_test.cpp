// Similarity self-join through the C++ host mirror (gpu::EmbeddingIndex::SearchPairs).
//   ./pairs_mirror_test            (needs a GPU)      ./pairs_mirror_test --no-gpu   (compiles and links only)
#include <cstdio>
#include <cstring>

#include "nornicdb_b200/host/nornic_cuda.hpp"

using namespace nornic;

int main(int argc, char **argv) {
    if (argc > 1 && std::strcmp(argv[1], "--no-gpu") == 0) {
        std::printf("pairs mirror ok\n");
        return 0;
    }
    int failures = 0;
    auto expect = [&](bool ok, const char *what) {
        if (!ok) { std::printf("FAIL: %s\n", what); ++failures; }
    };
    gpu::EmbeddingIndex ix(4);
    ix.Add("person-a", {1, 0, 0, 0});
    ix.Add("doc-b", {0.9f, 0.1f, 0, 0});
    ix.Add("person-c", {0, 1, 0, 0});
    ix.Add("person-d", {1, 0, 0, 0});
    const uint64_t PERSON = 1, DOC = 2;
    ix.SetRowTags(0, {PERSON, DOC, PERSON, PERSON});
    auto p = ix.SearchPairs(0.9f);
    // a-b, a-d, b-d reach 0.9; c is orthogonal to all
    expect(p.size() == 3, "three pairs reach 0.9");
    expect(p.size() == 3 && p[0].A == "person-a" && p[0].B == "person-d" && p[1].A == "person-a" && p[1].B == "doc-b",
           "pairs of the lowest row first, best first");
    expect(p.size() == 3 && p[2].A == "doc-b" && p[2].B == "person-d", "each pair once, under its lower row");
    const NkFilter persons{PERSON, 0, 0};
    auto f = ix.SearchPairs(0.9f, &persons);
    expect(f.size() == 1 && f[0].A == "person-a" && f[0].B == "person-d", "filter applies to both sides");
    auto s = ix.SearchPairs(-1.0f, nullptr, 1);
    expect(s.size() == 6, "threshold -1 in one-row stripes: all 4*3/2 pairs");
    std::printf(failures ? "%d FAILURES\n" : "pairs mirror ok\n", failures);
    return failures ? 1 : 0;
}
