// merkle_update.cuh -- the plan of a batched Merkle update (MerkleTree::update / check_update, R/merkle_tree/mod.rs:627-725):
// which nodes k new leaf digests touch, where each touched node's children are, and where its new value goes.
//
// Levels are numbered from the root: level l (0 <= l < h) holds the 2^l inner nodes at heap positions [2^l - 1, 2^(l+1) - 1),
// level h the n = 2^h leaves.  U[0 .. m) is the sorted set of distinct updated leaf indexes (the last occurrence of an index
// supplies its digest).  A node p of level l is touched when some U[i] >> (h - l) == p; its OWNER is the first such i.
//
// New values live in scratch, Σ_l min(k, 2^l) elements: level l has width z_l = min(k, 2^l) slots from off[l] on.  A DENSE
// level (2^l <= k) is indexed by node (slot = p); a sparse one by owner (slot = i < m <= k).  A level's kernel runs one
// candidate per slot: candidate c is node c (dense) or U position c (sparse) and hashes only when that node is touched, so
// every touched node is hashed exactly once and no per-level list has to be built.  Lookups are binary searches in U.
//
// Everything here is CPB_HD: tests/host/merkle_update_shim.cpp runs it on the CPU against a Python model.
#pragma once
#include "ptx.cuh"

#include <algorithm>
#include <vector>

namespace cpb {

constexpr int kUpdMaxLevels = 64;   // h <= 63 (n is a size_t power of two)

struct UpdPlan {
    const u64* U = nullptr;         // sorted distinct leaf indexes, m of them
    const u64* m = nullptr;         // device word: the number of distinct in-range indexes
    int h = 0;
    u64 k = 0;                      // number of (index, digest) pairs given
    u64 off[kUpdMaxLevels + 2] = {};   // scratch offset of level l (elements); off[h + 1] = total
};

CPB_HD bool upd_dense(int l, u64 k) { return (1ull << l) <= k; }
CPB_HD u64 upd_width(int l, u64 k) { return upd_dense(l, k) ? (1ull << l) : k; }

// Scratch offsets of levels 0 .. h and the total (off[h + 1]).
CPB_HD void upd_offsets(int h, u64 k, u64* off) {
    off[0] = 0;
    for (int l = 0; l <= h; l++) off[l + 1] = off[l] + upd_width(l, k);
}

// First i in [0, m) with U[i] >= key (m when none).
CPB_HD u64 upd_lower_bound(const u64* U, u64 m, u64 key) {
    u64 lo = 0, hi = m;
    while (lo < hi) {
        const u64 mid = lo + ((hi - lo) >> 1);
        if (U[mid] < key) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

struct UpdSite {
    bool touched = false;
    u64 node = 0;     // index within the level
    u64 owner = 0;    // first U position under the node
    u64 slot = 0;     // scratch slot within the level
};

// Candidate `cand` (< upd_width(l, k)) of level l (0 <= l <= h).
CPB_HD UpdSite upd_site(const u64* U, u64 m, int h, int l, u64 k, u64 cand) {
    UpdSite S;
    const int s = h - l;
    if (upd_dense(l, k)) {
        S.node = cand;
        S.owner = upd_lower_bound(U, m, cand << s);
        S.touched = S.owner < m && (U[S.owner] >> s) == cand;
    } else {
        S.owner = cand;
        S.touched = cand < m && (cand == 0 || (U[cand] >> s) != (U[cand - 1] >> s));
        if (S.touched) S.node = U[cand] >> s;
    }
    S.slot = upd_dense(l, k) ? S.node : S.owner;
    return S;
}

// Children (at level l + 1) of a touched node of level l < h: which are touched, and their slots when they are.
struct UpdKids {
    bool lt = false, rt = false;
    u64 lslot = 0, rslot = 0;
};
CPB_HD UpdKids upd_kids(const u64* U, u64 m, int h, int l, u64 k, const UpdSite& S) {
    UpdKids K;
    const int s = h - l - 1;                                   // shift of the child level
    const u64 left = 2 * S.node, right = left + 1;
    K.lt = ((U[S.owner] >> s) & 1) == 0;                       // the owner is the first index under the node
    const u64 j = K.lt ? upd_lower_bound(U, m, right << s) : S.owner;
    K.rt = j < m && (U[j] >> s) == right;
    const bool dense = upd_dense(l + 1, k);
    K.lslot = dense ? left : S.owner;
    K.rslot = dense ? right : j;
    return K;
}

// Where the current value of child `node` (level l + 1) of a touched node of level l is, for digests of W words: the scratch when
// the child is touched too, the caller's tree otherwise (its leaf array below level h - 1, its heap-ordered inner nodes above).
template <int W, class T>
CPB_HD T* upd_child_at(const UpdPlan& X, int l, bool touched, u64 slot, u64 node, T* scratch, T* leaf_nodes, T* nodes) {
    if (touched) return scratch + W * (X.off[l + 1] + slot);
    if (l + 1 == X.h) return leaf_nodes + W * node;
    return nodes + W * (((1ull << (l + 1)) - 1) + node);
}

// The candidate of level l - 1 that is the parent of node p of level l (l > 0).
CPB_HD u64 upd_parent_cand(const u64* U, u64 m, int h, int l, u64 k, u64 p) {
    const u64 q = p >> 1;
    return upd_dense(l - 1, k) ? q : upd_lower_bound(U, m, q << (h - l + 1));
}

// Flat commit index t < off[h + 1] -> its level.
CPB_HD int upd_level_of(const u64* off, int h, u64 t) {
    int l = 0;
    while (l < h && t >= off[l + 1]) l++;
    return l;
}

// ---- host forms: which tree nodes the device code reads and writes, by index arithmetic on the distinct sorted indexes.
// Positions are in one array of 2n - 1 elements: leaf c at c, inner node at heap position q at n + q.
// reads: the untouched children of touched inner nodes; writes: every touched node (leaves and inner nodes).
inline void upd_host_sets(const std::vector<u64>& uniq, int h, std::vector<u64>& reads, std::vector<u64>& writes) {
    const u64 n = 1ull << h;
    reads.clear();
    writes.clear();
    std::vector<u64> cur = uniq, up;
    for (int l = h; l >= 0; l--) {                             // cur: touched nodes of level l, sorted and distinct
        const u64 base = l == h ? 0 : n + ((1ull << l) - 1);
        for (size_t j = 0; j < cur.size(); j++) {
            writes.push_back(base + cur[j]);
            const u64 sib = cur[j] ^ 1;
            const bool sib_touched = (j > 0 && cur[j - 1] == sib) || (j + 1 < cur.size() && cur[j + 1] == sib);
            if (l > 0 && !sib_touched) reads.push_back(base + sib);
        }
        up.clear();
        for (u64 p : cur)
            if (up.empty() || up.back() != (p >> 1)) up.push_back(p >> 1);
        cur.swap(up);
    }
}

}  // namespace cpb
