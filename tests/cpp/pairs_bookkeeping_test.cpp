// SimilarPairs' bookkeeping in the C++ host mirror, without a GPU: the mirror is linked against a stand-in of the few C calls
// it makes here, which records what nk_pairs_remap is handed.  After Add (new and existing ids), AddBatch, Remove, SetRowTags
// and SetRowValues the row map must say, for each row, which row of the last join its contents came from (NK_ROW_NEW for new
// contents); a change of threshold, filter, window or gap, or a Deserialize, must rebuild instead.
//   ./pairs_bookkeeping_test
#include <cstdio>
#include <cstring>

#include "nornicdb_b200/host/nornic_cuda.hpp"

// ---- the stand-in: rows are counted, pairs are never found ----------------------------------------------------------------
struct NkIndex { uint64_t rows = 0; };
static std::vector<uint32_t> g_src;   // the src_of_row of the last nk_pairs_remap
static uint64_t g_n_old = 0, g_remaps = 0, g_joins = 0;
extern "C" {
NkIndex *nk_index_create(const int *, int, uint32_t, int, int) { return new NkIndex(); }
void nk_index_release(NkIndex *ix) { delete ix; }
const char *nk_last_error(void) { return "stand-in"; }
uint64_t nk_index_rows(const NkIndex *ix) { return ix->rows; }
int nk_index_append(NkIndex *ix, const void *, uint64_t n) { ix->rows += n; return 0; }
int nk_index_update_row(NkIndex *, uint64_t, const void *) { return 0; }
int nk_index_remove_swap(NkIndex *ix, uint64_t) { --ix->rows; return 0; }
int nk_index_upload(NkIndex *ix, const void *, uint64_t n) { ix->rows = n; return 0; }
int nk_index_read_rows(NkIndex *, uint64_t, uint64_t, void *) { return 0; }
int nk_index_set_row_tags(NkIndex *, uint64_t, const uint64_t *, uint64_t) { return 0; }
int nk_index_set_row_values(NkIndex *, uint64_t, const uint64_t *, uint64_t) { return 0; }
int nk_index_set_path(NkIndex *, int) { return 0; }
int nk_search_pairs_windowed(NkIndex *, uint64_t, uint64_t n_rows, float, const NkFilter *, const NkWindow *, uint64_t, uint64_t,
                             uint64_t *off, uint32_t *, float *, uint64_t *total) {
    ++g_joins;
    for (uint64_t r = 0; r <= n_rows; ++r) off[r] = 0;
    *total = 0;
    return 0;
}
int nk_pairs_remap(NkIndex *ix, float, const NkFilter *, const NkWindow *, uint64_t, uint64_t n_old, const uint32_t *src,
                   const uint64_t *, const uint32_t *, const float *, uint64_t, uint64_t *off, uint32_t *, float *, uint64_t *total,
                   uint64_t *, uint64_t *) {
    ++g_remaps;
    g_n_old = n_old;
    g_src.assign(src, src + ix->rows);
    for (uint64_t r = 0; r <= ix->rows; ++r) off[r] = 0;
    *total = 0;
    return 0;
}
}

using namespace nornic;

int main() {
    int failures = 0;
    auto expect = [&](bool ok, const char *what) {
        if (!ok) { std::printf("FAIL: %s\n", what); ++failures; }
    };
    const uint32_t NEW = NK_ROW_NEW;
    gpu::EmbeddingIndex ix(2);
    for (int i = 0; i < 6; ++i) ix.Add("n" + std::to_string(i), {1.0f, (float)i});
    const NkFilter f{0, 2, 0};
    ix.SimilarPairs(0.5f, &f);
    expect(g_joins == 1 && ix.PairsRebuilds() == 1 && g_remaps == 0, "the first call joins");
    ix.Add("n6", {0, 1});                               // append: row 6
    ix.Add("n2", {0, 1});                               // rewrite of row 2
    ix.Remove("n0");                                    // row 6 (new) moves into row 0
    ix.Remove("n4");                                    // row 5 moves into row 4
    ix.SetRowTags(0, {0, 1, 0, 0, 0});                  // row 1 retagged; the others unchanged
    ix.SetRowValues(3, {7});                            // row 3 re-valued
    ix.SetRowValues(0, {0});                            // row 0: the same key (0) again
    ix.SimilarPairs(0.5f, &f);
    expect(g_remaps == 1 && ix.PairsRebuilds() == 1, "kept current by a remap");
    expect(g_n_old == 6, "the remap is handed the join's row count");
    const std::vector<uint32_t> want{NEW, NEW, NEW, NEW, 5};
    expect(g_src == want, "row map after append, rewrite, removals, a retag and a re-value");
    ix.AddBatch({"a", "b"}, {{1, 1}, {2, 2}});
    ix.Remove("n3");                                    // row 3: the last row ("b", new) moves into it
    ix.SimilarPairs(0.5f, &f);
    expect(g_remaps == 2 && g_n_old == 5, "a second remap from the join the first one left");
    const std::vector<uint32_t> want2{0, 1, 2, NEW, 4, NEW};
    expect(g_src == want2, "rows kept at their id after the last call, new rows NEW, the moved new row NEW");
    ix.SimilarPairs(0.5f, nullptr);
    expect(ix.PairsRebuilds() == 2 && g_remaps == 2, "a new filter rebuilds");
    const NkWindow w{1, 9};
    ix.SimilarPairs(0.5f, nullptr, &w);
    expect(ix.PairsRebuilds() == 3, "a new window rebuilds");
    ix.SimilarPairs(0.5f, nullptr, &w, 3);
    expect(ix.PairsRebuilds() == 4, "a new gap rebuilds");
    ix.SimilarPairs(0.6f, nullptr, &w, 3);
    expect(ix.PairsRebuilds() == 5, "a new threshold rebuilds");
    ix.SimilarPairs(0.6f, nullptr, &w, 3);
    expect(ix.PairsRebuilds() == 5 && g_remaps == 3, "the same arguments remap");
    const std::vector<uint32_t> want3{0, 1, 2, 3, 4, 5};
    expect(g_src == want3, "nothing changed: every row kept");
    ix.Deserialize(ix.Serialize());
    ix.SimilarPairs(0.6f, nullptr, &w, 3);
    expect(ix.PairsRebuilds() == 6, "a Deserialize rebuilds");
    std::printf(failures ? "%d FAILURES\n" : "pairs bookkeeping ok\n", failures);
    return failures ? 1 : 0;
}
