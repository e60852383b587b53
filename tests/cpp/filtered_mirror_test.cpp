// Per-query tag filters through the C++ host mirror (gpu::EmbeddingIndex::SetRowTags / SearchBatchFiltered).
//   ./filtered_mirror_test            (needs a GPU)      ./filtered_mirror_test --no-gpu   (compiles and links only)
#include <cstdio>
#include <cstring>

#include "nornicdb_b200/host/nornic_cuda.hpp"

using namespace nornic;

int main(int argc, char **argv) {
    if (argc > 1 && std::strcmp(argv[1], "--no-gpu") == 0) {
        std::printf("filtered mirror ok\n");
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
    const std::vector<float> q = {1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0};
    const std::vector<NkFilter> f = {{0, 0, 0}, {DOC, 0, 0}, {0, PERSON, 0}};
    auto r = ix.SearchBatchFiltered(q, f, 3, 3);
    expect(r.size() == 3, "one result list per query");
    expect(r[0].size() == 3 && r[0][0].ID == "person-a" && r[0][1].ID == "doc-b", "no filter: every row");
    expect(r[1].size() == 1 && r[1][0].ID == "doc-b", "all_of: only the tagged row, the rest padding");
    expect(r[2].size() == 1 && r[2][0].ID == "doc-b", "none_of: the excluded label never comes back");
    std::printf(failures ? "%d FAILURES\n" : "filtered mirror ok\n", failures);
    return failures ? 1 : 0;
}
