// Range search through the C++ host mirror (gpu::EmbeddingIndex::SearchRange).
//   ./range_mirror_test            (needs a GPU)      ./range_mirror_test --no-gpu   (compiles and links only)
#include <cstdio>
#include <cstring>

#include "nornicdb_b200/host/nornic_cuda.hpp"

using namespace nornic;

int main(int argc, char **argv) {
    if (argc > 1 && std::strcmp(argv[1], "--no-gpu") == 0) {
        std::printf("range mirror ok\n");
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
    const uint64_t PERSON = 1, DOC = 2;
    ix.SetRowTags(0, {PERSON, DOC, PERSON});
    const std::vector<float> q = {1, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0};
    auto r = ix.SearchRange(q, {0.9f, -1.0f, 2.0f}, {}, 3);
    expect(r.size() == 3, "one result list per query");
    expect(r[0].size() == 2 && r[0][0].ID == "person-a" && r[0][1].ID == "doc-b", "threshold 0.9: the two close rows, best first");
    expect(r[1].size() == 3, "threshold -1: every row");
    expect(r[2].empty(), "threshold above 1: nothing");
    auto f = ix.SearchRange(q, {-1.0f, -1.0f, -1.0f}, {{PERSON, 0, 0}, {DOC, 0, 0}, {0, PERSON, 0}}, 3);
    expect(f[0].size() == 2 && f[0][0].ID == "person-a" && f[0][1].ID == "person-c", "all_of PERSON");
    expect(f[1].size() == 1 && f[1][0].ID == "doc-b", "all_of DOC");
    expect(f[2].size() == 1 && f[2][0].ID == "doc-b", "none_of PERSON");
    std::printf(failures ? "%d FAILURES\n" : "range mirror ok\n", failures);
    return failures ? 1 : 0;
}
