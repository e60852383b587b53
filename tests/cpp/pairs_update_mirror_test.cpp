// The self-join kept current through the C++ host mirror (gpu::EmbeddingIndex::SimilarPairs and PairsOfNodes).
//   ./pairs_update_mirror_test            (needs a GPU)      ./pairs_update_mirror_test --no-gpu   (compiles and links only)
// After every change (Add of a new node, Add of an existing one, Remove, SetRowTags, SetRowValues) the maintained join must
// equal the join of a fresh index holding the same rows, tags and value keys, without a rebuild; PairsOfNodes of a changed
// node must be that join's pairs of the node.
#include <cstdio>
#include <cstring>
#include <set>
#include <tuple>

#include "nornicdb_b200/host/nornic_cuda.hpp"

using namespace nornic;

static uint64_t lcg = 12345;
static float rnd() {
    lcg = lcg * 6364136223846793005ull + 1442695040888963407ull;
    return (float)((lcg >> 33) % 2001) / 1000.0f - 1.0f;
}

static std::vector<float> vec(int d, const std::vector<float> *near = nullptr) {
    std::vector<float> v(d);
    for (int i = 0; i < d; ++i) v[i] = near ? (*near)[i] + 0.05f * rnd() : rnd();
    return v;
}

// A fresh index with the same rows (Serialize / Deserialize keeps the row order), tags and value keys.
static std::vector<gpu::SimilarPair> fresh_join(gpu::EmbeddingIndex &ix, int d, float t, const NkFilter *f, const NkWindow *w, uint64_t gap) {
    gpu::EmbeddingIndex fresh(d);
    fresh.Deserialize(ix.Serialize());
    if (fresh.Count()) {
        fresh.SetRowTags(0, ix.RowTags());
        fresh.SetRowValues(0, ix.RowValues());
    }
    return fresh.SimilarPairs(t, f, w, gap);
}

static bool same(const std::vector<gpu::SimilarPair> &a, const std::vector<gpu::SimilarPair> &b) {
    if (a.size() != b.size()) return false;
    for (size_t i = 0; i < a.size(); ++i)
        if (a[i].A != b[i].A || a[i].B != b[i].B || std::memcmp(&a[i].Score, &b[i].Score, 4) != 0) return false;
    return true;
}

int main(int argc, char **argv) {
    if (argc > 1 && std::strcmp(argv[1], "--no-gpu") == 0) {
        std::printf("pairs update mirror ok\n");
        return 0;
    }
    int failures = 0;
    auto expect = [&](bool ok, const char *what) {
        if (!ok) { std::printf("FAIL: %s\n", what); ++failures; }
    };
    const int d = 32, n = 600;
    gpu::EmbeddingIndex ix(d);
    std::vector<std::vector<float>> centres;
    for (int c = 0; c < 30; ++c) centres.push_back(vec(d));
    for (int i = 0; i < n; ++i) ix.Add("n" + std::to_string(i), vec(d, &centres[i % 30]));
    std::vector<uint64_t> tags(n), keys(n);
    for (int i = 0; i < n; ++i) { tags[i] = (uint64_t)(i % 3); keys[i] = 1 + (uint64_t)(i * 7 % 100); }
    ix.SetRowTags(0, tags);
    ix.SetRowValues(0, keys);
    const float t = 0.9f;
    const NkFilter flt{0, 2, 0};  // rows tagged 2 are refused
    const NkWindow win{5, 95};
    struct Args { const NkFilter *f; const NkWindow *w; uint64_t gap; const char *name; };
    for (const Args &a : {Args{nullptr, nullptr, NK_NO_GAP, "plain"}, Args{&flt, &win, 20, "filter, window and band"}}) {
        auto p0 = ix.SimilarPairs(t, a.f, a.w, a.gap);
        expect(!p0.empty(), "the join has pairs");
        expect(same(p0, fresh_join(ix, d, t, a.f, a.w, a.gap)), "first call: the fresh join");
        const uint64_t rebuilds = ix.PairsRebuilds();
        int step = 0;
        auto check_step = [&](const char *what, const std::string &changed) {
            ++step;
            auto p = ix.SimilarPairs(t, a.f, a.w, a.gap);
            auto want = fresh_join(ix, d, t, a.f, a.w, a.gap);
            if (!same(p, want)) std::printf("  %s / %s: %zu pairs, fresh join %zu\n", a.name, what, p.size(), want.size());
            expect(same(p, want), what);
            expect(ix.PairsRebuilds() == rebuilds, "kept current without a rebuild");
            if (changed.empty() || !ix.Has(changed)) return;
            std::set<std::tuple<std::string, std::string, uint32_t>> mine, of_join;
            for (auto &e : ix.PairsOfNodes({changed}, t, a.f, a.w, a.gap)) {
                expect(e.A == changed, "PairsOfNodes: the listed node first");
                uint32_t b;
                std::memcpy(&b, &e.Score, 4);
                mine.insert({e.A, e.B, b});
            }
            for (auto &e : p)
                if (e.A == changed || e.B == changed) {
                    uint32_t b;
                    std::memcpy(&b, &e.Score, 4);
                    of_join.insert({changed, e.A == changed ? e.B : e.A, b});
                }
            expect(mine == of_join, "PairsOfNodes: the join's pairs of the node");
        };
        ix.Add("new" + std::to_string(step), vec(d, &centres[3]));
        check_step("Add of a new node", "new0");
        ix.Add("n7", vec(d, &centres[11]));
        check_step("Add of an existing node (rewrite)", "n7");
        ix.Remove("n10");  // the last node moves into row 10
        ix.Remove("n3");
        check_step("Remove", ix.Has("new0") ? "new0" : "");
        std::vector<uint64_t> tg = ix.RowTags();
        tg[5] = 2;
        tg[9] = 0;
        ix.SetRowTags(0, tg);
        check_step("SetRowTags", "n5");
        std::vector<uint64_t> kv = ix.RowValues();
        kv[20] = 90;
        kv[21] = 0;
        ix.SetRowValues(0, kv);
        check_step("SetRowValues", "n20");
        ix.AddBatch({"b0", "b1", "n40"}, {vec(d, &centres[0]), vec(d, &centres[1]), vec(d, &centres[2])});
        check_step("AddBatch", "b1");
        ix.SimilarPairs(t + 0.01f, a.f, a.w, a.gap);
        expect(ix.PairsRebuilds() == rebuilds + 1, "a new threshold rebuilds");
        auto s1 = ix.SimilarPairs(t, a.f, a.w, a.gap, 100);  // rebuilt again, in stripes of 100 rows
        expect(same(s1, fresh_join(ix, d, t, a.f, a.w, a.gap)), "a join built in stripes");
    }
    std::printf(failures ? "%d FAILURES\n" : "pairs update mirror ok\n", failures);
    return failures ? 1 : 0;
}
