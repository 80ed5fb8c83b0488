// CPU run of the Merkle update plan (crypto_primitives_b200/csrc/merkle_update.cuh) for tests/test_merkle_update_host.py: the steps of
// cpb_merkle_update.cu done sequentially with the same plan functions, over one-word toy digests and a toy two-to-one hash.  The
// levels above `lt` (the team launch) are processed in a seeded random order with the device's arrival counters, as any
// interleaving of CTAs would.  Not part of the product.
#include "../../crypto_primitives_b200/csrc/merkle_update.cuh"

#include <algorithm>
#include <cstdint>
#include <random>
#include <utility>
#include <vector>
using namespace cpb;

extern "C" uint64_t host_upd_toy_hash(uint64_t a, uint64_t b) { return a * 0x9E3779B97F4A7C15ull + b * 0xC2B2AE3D27D4EB4Full + 1; }

extern "C" void host_upd_offsets(int h, uint64_t k, uint64_t* off) { upd_offsets(h, k, off); }

// Returns `applied`; *hashes = two-to-one hashes done, *scratch = scratch elements used.
extern "C" int host_upd_run(const uint64_t* idx, const uint64_t* digests, uint64_t k, int h, int lt, uint64_t* leaf_nodes, uint64_t* nodes,
                            const uint64_t* asserted, uint64_t seed, uint64_t* hashes, uint64_t* scratch_elems) {
    const u64 n = 1ull << h;
    UpdPlan X;
    X.h = h;
    X.k = k;
    upd_offsets(h, k, X.off);
    *hashes = 0;
    *scratch_elems = X.off[h + 1];
    // plan: stable sort of (key, position), keep the last of each in-range run
    std::vector<std::pair<u64, unsigned>> kv(k);
    for (u64 j = 0; j < k; j++) kv[j] = {idx[j] < n ? idx[j] : n, (unsigned)j};
    std::stable_sort(kv.begin(), kv.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
    std::vector<u64> U;
    std::vector<u64> scratch(X.off[h + 1] + 1, 0xDEADull);
    for (u64 j = 0; j < k; j++) {
        if (!(kv[j].first < n && (j + 1 == k || kv[j + 1].first != kv[j].first))) continue;
        const u64 i = U.size();
        U.push_back(kv[j].first);
        scratch[X.off[h] + (upd_dense(h, k) ? kv[j].first : i)] = digests[kv[j].second];
    }
    const u64 m = U.size();
    const u64* Up = U.data();
    auto child = [&](int l, bool touched, u64 slot, u64 node) -> u64 {
        if (touched) return scratch[X.off[l + 1] + slot];
        if (l + 1 == h) return leaf_nodes[node];
        return nodes[((1ull << (l + 1)) - 1) + node];
    };
    auto hash_site = [&](int l, const UpdSite& S) {
        const UpdKids K = upd_kids(Up, m, h, l, k, S);
        scratch[X.off[l] + S.slot] = host_upd_toy_hash(child(l, K.lt, K.lslot, 2 * S.node), child(l, K.rt, K.rslot, 2 * S.node + 1));
        ++*hashes;
    };
    const int l_grid_end = lt >= 0 ? lt + 1 : 0;
    for (int l = h - 1; l >= l_grid_end; l--)
        for (u64 c = 0; c < upd_width(l, k); c++) {
            const UpdSite S = upd_site(Up, m, h, l, k, c);
            if (S.touched) hash_site(l, S);
        }
    if (lt >= 0) {
        std::vector<unsigned> arrivals(X.off[lt] + 1, 0);
        std::vector<std::pair<int, UpdSite>> work;
        for (u64 c = 0; c < upd_width(lt, k); c++) {
            const UpdSite S = upd_site(Up, m, h, lt, k, c);
            if (S.touched) work.push_back({lt, S});
        }
        std::mt19937_64 rng(seed);
        while (!work.empty()) {
            const size_t pick = rng() % work.size();
            const auto [l, S] = work[pick];
            work[pick] = work.back();
            work.pop_back();
            hash_site(l, S);
            if (l == 0) continue;
            const u64 pc = upd_parent_cand(Up, m, h, l, k, S.node);
            const UpdSite PS = upd_site(Up, m, h, l - 1, k, pc);
            const UpdKids PK = upd_kids(Up, m, h, l - 1, k, PS);
            const unsigned need = (PK.lt ? 1u : 0u) + (PK.rt ? 1u : 0u);
            if (++arrivals[X.off[l - 1] + PS.slot] == need) work.push_back({l - 1, PS});
        }
    }
    // commit
    const u64 root = m ? scratch[X.off[0]] : nodes[0];
    const bool ok = !asserted || root == *asserted;
    if (!ok || m == 0) return ok;
    for (u64 t = 0; t < X.off[h + 1]; t++) {
        const int l = upd_level_of(X.off, h, t);
        const UpdSite S = upd_site(Up, m, h, l, k, t - X.off[l]);
        if (!S.touched) continue;
        if (l == h) leaf_nodes[S.node] = scratch[t];
        else nodes[((1ull << l) - 1) + S.node] = scratch[t];
    }
    return 1;
}

// upd_host_sets over the distinct sorted indexes: writes *nr / *nw and, when the buffers are given, the positions.
extern "C" void host_upd_sets(const uint64_t* uniq, uint64_t m, int h, uint64_t* reads, uint64_t* nr, uint64_t* writes, uint64_t* nw) {
    std::vector<u64> u(uniq, uniq + m), r, w;
    upd_host_sets(u, h, r, w);
    *nr = r.size();
    *nw = w.size();
    if (reads) std::copy(r.begin(), r.end(), reads);
    if (writes) std::copy(w.begin(), w.end(), writes);
}
