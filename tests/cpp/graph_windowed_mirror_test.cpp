// A windowed k-NN graph through the C++ host mirror (gpu::EmbeddingIndex::SimilarGraph(k, filters, windows)): a time-local
// graph (each node's list holds only nodes within a day of its own timestamp), kept current across SetRowValues (a node
// moved in time), Remove, Add and a changed window: after each sequence the graph equals one built from scratch with the same
// value keys and windows, and the index itself never rebuilt it.
//   ./graph_windowed_mirror_test            (needs a GPU)      ./graph_windowed_mirror_test --no-gpu   (compiles and links only)
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

static const uint64_t HOUR = 3600, DAY = 24 * HOUR;

// each node's band: its own key +- one day (a node without a value, key 0, gets the window that admits no node)
static std::vector<NkWindow> bands(const std::vector<uint64_t> &keys) {
    std::vector<NkWindow> w(keys.size());
    for (size_t r = 0; r < keys.size(); ++r)
        w[r] = keys[r] ? NkWindow{keys[r] > DAY ? keys[r] - DAY : 1, keys[r] + DAY} : NkWindow{~0ull, 0};
    return w;
}

int main(int argc, char **argv) {
    if (argc > 1 && std::strcmp(argv[1], "--no-gpu") == 0) {
        std::printf("graph windowed mirror ok\n");
        return 0;
    }
    int failures = 0;
    auto expect = [&](bool ok, const std::string &what) {
        if (!ok) { std::printf("FAIL: %s\n", what.c_str()); ++failures; }
    };
    const int D = 64, K = 5;
    uint64_t state = 4242;
    auto next = [&]() { state = state * 6364136223846793005ull + 1442695040888963407ull; return state >> 33; };
    auto vec = [&]() {
        std::vector<float> v(D);
        for (auto &x : v) x = (float)(next() % 2001) / 1000.0f - 1.0f;
        return v;
    };
    const uint64_t T0 = 1000 * DAY;
    gpu::EmbeddingIndex ix(D);
    std::vector<std::vector<float>> seed;
    for (int i = 0; i < 400; ++i) { seed.push_back(vec()); ix.Add("n" + std::to_string(i), seed.back()); }
    // timestamps over 30 days; the last three nodes alone 100 days later (short lists), node 7 without a value
    std::vector<uint64_t> keys(400);
    for (int i = 0; i < 400; ++i) keys[i] = i < 397 ? T0 + next() % (30 * DAY) : T0 + 100 * DAY + (uint64_t)i;
    keys[7] = 0;
    ix.SetRowValues(0, keys);
    auto g0 = ix.SimilarGraph(K, {}, bands(ix.RowValues()));
    expect(g0.size() == 400 && ix.GraphRebuilds() == 1, "the first call builds the graph");
    expect(g0[399].size() == 2 && g0[7].empty(), "a lone day's lists are short, a node without a value has none");
    auto check = [&](const std::string &what, const std::vector<NkWindow> &windows) {
        auto g = ix.SimilarGraph(K, {}, windows);
        gpu::EmbeddingIndex fresh(D);
        fresh.Deserialize(ix.Serialize());
        fresh.SetRowValues(0, ix.RowValues());
        auto r = fresh.SimilarGraph(K, {}, windows);
        expect(fresh.GraphRebuilds() == 1 && (int)g.size() == ix.Count() && same(g, r), what + " equals a rebuild");
        expect(ix.GraphRebuilds() == 1, what + ": no rebuild");
    };
    // nodes moved in time: into the lone day, a week on, and to no value
    ix.SetRowValues(20, {T0 + 100 * DAY});
    ix.SetRowValues(21, {T0 + 7 * DAY + 5 * HOUR});
    ix.SetRowValues(22, {0});
    check("SetRowValues", bands(ix.RowValues()));
    // Remove, and Add: a near copy of a lone-day node stamped into its day, a rewrite in place, a new node in the bulk
    ix.Remove("n10");
    ix.Add("a0", seed[398]);
    ix.SetRowValues((uint64_t)ix.Count() - 1, {T0 + 100 * DAY + 2 * HOUR});
    ix.Add("n33", vec());
    ix.Add("a1", vec());
    ix.SetRowValues((uint64_t)ix.Count() - 1, {T0 + 3 * DAY});
    ix.Remove("n0");
    check("Remove / Add", bands(ix.RowValues()));
    // one node's window widens to the whole range, another's narrows to an hour
    auto w = bands(ix.RowValues());
    w[5] = NkWindow{1, ~0ull};
    w[6] = NkWindow{ix.RowValues()[6], ix.RowValues()[6] + HOUR};
    check("window change", w);
    for (int i = 0; i < 20; ++i) {
        ix.Remove("n" + std::to_string(40 + 7 * i));
        ix.Add("b" + std::to_string(i), vec());
        ix.SetRowValues((uint64_t)ix.Count() - 1, {T0 + (uint64_t)i * DAY});
    }
    w = bands(ix.RowValues());
    w[5] = NkWindow{1, ~0ull};
    check("interleaved Add / Remove / SetRowValues", w);
    std::printf(failures ? "%d FAILURES\n" : "graph windowed mirror ok\n", failures);
    return failures ? 1 : 0;
}
