// mstep_rows.h — row layout of the tensor M-step's feature operand (host side, plain C++).
//
// Operand row r of feature tile mt is the product z_a * z_b of two factors: a dimension of the centred / scaled event,
// or the ones pseudo-dimension (a linear statistic z_i is z_i * 1, the constant row 1 * 1).  The consumer thread
// (warp w of the tile's warpgroup, lane group gid = lane / 4) builds the wgmma A fragments of its four rows
//     mt * 128 + h * 64 + 16 w + gid + 8 s        (h, s in {0, 1}; slot = 2 h + s)
// itself, from the z tile in shared memory.  The four rows share their first factor a, so a thread loads 5 rows of the
// z tile (a and the four b) per sub-tile.
//
// Which feature tile a statistic belongs to is fixed (mstep_stat_tiles): the tiles' accumulation chains are staggered,
// so the tile decides where a statistic's FP32 partial sums are rounded.  The assignment is the one of the earlier
// layout, in which four builder warps evaluated the canonical rows [1, z'_a, z'_a^2, z'_a z'_(a+d)] of a rotated event.
// Inside a tile the statistics are packed greedily into 32 groups of at most 4 that share a factor, and the groups are
// placed so that the rows the 8 lane groups of a warp load at once fall into different bank groups of the SWIZZLE_128B
// z tile (16-byte chunk c of row d sits at chunk c ^ (d & 7)).  Codes kRowOne + rho name row rho of a 1 KB block of ones
// with the same swizzle (every row reads 1.0): rho is chosen to fill the least used bank group.
// tests/test_mstep_rowmap.py checks the layout at every D.
#pragma once
#include <algorithm>
#include <array>
#include <vector>

namespace gmm {

constexpr int kRowOne = 32;

struct MRow {
    int f, i, j;   // packed statistic (-1: unused row) and its dimensions (-1: none), for the un-scaling
    int a, b;      // operand factors: dimension, or kRowOne + rho
};

inline int mstep_feat2(int D, int i, int j) { return 1 + D + i * (i + 1) / 2 + j; }

// Feature tiles of the layout (128 rows each).
inline int mstep_tiles(int D) {
    const int S = D / 4, rpp = 1 + 2 * S + S * (D / 2), rows = 4 * ((rpp + 7) / 8) * 8;
    return (rows + 127) / 128;
}

// Feature tile of every packed statistic (F = 1 + D + D (D + 1) / 2 entries).
inline std::vector<int> mstep_stat_tiles(int D) {
    const int S = D / 4, half = D / 2, rpp = 1 + 2 * S + S * half, cpp = (rpp + 7) / 8;
    std::vector<int> tile(1 + D + D * (D + 1) / 2, -1);
    for (int row = 0; row < 4 * cpp * 8; row++) {
        const int p = row / (cpp * 8), r = row % (cpp * 8);
        int f = -1;
        if (r >= rpp) continue;
        if (r == 0) f = p == 0 ? 0 : -1;
        else if (r <= S) f = 1 + (r - 1 + p * S) % D;
        else {
            int a, b;
            if (r <= 2 * S) a = b = r - 1 - S;
            else { const int t = r - 1 - 2 * S; a = t / half; b = (a + 1 + t % half) % D; }
            const int ta = (a + p * S) % D, tb = (b + p * S) % D;
            if (!(a != b && (b - a + D) % D == half && ta >= half)) f = mstep_feat2(D, std::max(ta, tb), std::min(ta, tb));
        }
        if (f >= 0) tile[f] = row / 128;
    }
    return tile;
}

// [mstep_tiles(D) * 128] rows.
inline std::vector<MRow> mstep_row_layout(int D) {
    const int MT = mstep_tiles(D);
    const std::vector<int> tile = mstep_stat_tiles(D);
    std::vector<MRow> out((size_t)MT * 128, MRow{-1, -1, -1, kRowOne, kRowOne});
    constexpr int ONE = -1;                                  // factor index of the ones pseudo-dimension in the packing
    struct Item { int f, i, j, o0, o1; };                    // statistic, dimensions, candidate shared factors (o1 = -2: none)
    auto cls = [](int r) { return (r >> 1) & 3; };           // bank group of a z-tile row for an 8-event (32-byte) load
    for (int mt = 0; mt < MT; mt++) {
        std::vector<Item> items;
        for (int f = 0; f < (int)tile.size(); f++) {
            if (tile[f] != mt) continue;
            if (f == 0) items.push_back({f, -1, -1, ONE, -2});
            else if (f <= D) items.push_back({f, f - 1, -1, f - 1, ONE});
            else {
                int i = 0;
                while ((i + 1) * (i + 2) / 2 <= f - 1 - D) i++;
                const int j = f - 1 - D - i * (i + 1) / 2;
                items.push_back({f, i, j, i, i == j ? -2 : j});
            }
        }
        // greedy packing: close the factor with the fewest candidates, taking as many of them as fill whole groups of 4
        // (at least the ones no other open factor can take), preferring items whose other factor has many candidates
        std::vector<char> done(items.size(), 0), closed(D + 1, 0);
        std::vector<std::pair<int, std::vector<int>>> groups;     // (shared factor, items)
        for (;;) {
            std::vector<std::vector<int>> cand(D + 1);
            for (int k = 0; k < (int)items.size(); k++) {
                if (done[k]) continue;
                for (int o : {items[k].o0, items[k].o1})
                    if (o != -2 && !closed[o + 1]) cand[o + 1].push_back(k);
            }
            int best = -1;
            for (int g = 0; g <= D; g++)
                if (!cand[g].empty() && (best < 0 || cand[g].size() < cand[best].size())) best = g;
            if (best < 0) break;
            const int fac = best - 1;
            std::vector<int> forced, flex;
            for (int k : cand[best]) {
                const int other = items[k].o0 == fac ? items[k].o1 : items[k].o0;
                (other == -2 || closed[other + 1] ? forced : flex).push_back(k);
            }
            int m = (int)cand[best].size() / 4 * 4;
            if (m < (int)forced.size()) m = std::min((int)cand[best].size(), ((int)forced.size() + 3) / 4 * 4);
            auto other_cands = [&](int k) {
                const int other = items[k].o0 == fac ? items[k].o1 : items[k].o0;
                return (int)cand[other + 1].size();
            };
            std::stable_sort(flex.begin(), flex.end(), [&](int x, int y) { return other_cands(x) > other_cands(y); });
            std::vector<int> take = forced;
            for (int k = 0; k < (int)flex.size() && (int)take.size() < m; k++) take.push_back(flex[k]);
            for (size_t q = 0; q < take.size(); q += 4)
                groups.push_back({fac, std::vector<int>(take.begin() + q, take.begin() + std::min(take.size(), q + 4))});
            for (int k : take) done[k] = 1;
            closed[best] = 1;
        }
        if (groups.size() > 32) return {};                   // does not fit the tile (the caller reports it)
        std::stable_sort(groups.begin(), groups.end(), [](const auto& x, const auto& y) {
            return (x.first == ONE ? 1000 : x.first) < (y.first == ONE ? 1000 : y.first);
        });
        while (groups.size() < 32) groups.push_back({ONE, {}});
        // placement: group q -> warp q % 4 (the groups of one factor go to different warps, a warp's shared factors are
        // 8 consecutive ones: two per bank group), then per group the order of its rows over the 4 slots that adds the
        // fewest rows to the fullest bank group of each slot
        for (int w = 0; w < 4; w++) {
            std::array<std::vector<int>, 4> slot_rows;           // dimensions already loaded per slot by this warp
            std::array<std::array<int, 4>, 8> bsel{};            // [gid][slot] b factor (ONE: ones)
            std::array<std::array<int, 4>, 8> fsel{};            // [gid][slot] statistic
            std::array<int, 8> asel{};
            for (int gid = 0; gid < 8; gid++) {
                const auto& g = groups[gid * 4 + w];
                asel[gid] = g.first;
                std::array<int, 4> bs{ONE, ONE, ONE, ONE}, fs{-1, -1, -1, -1};
                for (size_t u = 0; u < g.second.size(); u++) {
                    const Item& it = items[g.second[u]];
                    fs[u] = it.f;
                    if (it.f == 0) bs[u] = ONE;
                    else if (it.j < 0) bs[u] = g.first == ONE ? it.i : ONE;
                    else bs[u] = g.first == it.i ? it.j : it.i;
                }
                auto waves = [&](const std::vector<int>& rows) {
                    int c[4] = {0, 0, 0, 0};
                    std::vector<int> seen;
                    for (int r : rows)
                        if (r != ONE && std::find(seen.begin(), seen.end(), r) == seen.end()) { seen.push_back(r); c[cls(r)]++; }
                    return *std::max_element(c, c + 4);
                };
                std::array<int, 4> perm{0, 1, 2, 3}, best_perm = perm;
                int best_cost = 1 << 30;
                do {
                    int cost = 0;
                    for (int s = 0; s < 4; s++) {
                        std::vector<int> rows = slot_rows[s];
                        rows.push_back(bs[perm[s]]);
                        cost += waves(rows);
                    }
                    if (cost < best_cost) { best_cost = cost; best_perm = perm; }
                } while (std::next_permutation(perm.begin(), perm.end()));
                for (int s = 0; s < 4; s++) {
                    slot_rows[s].push_back(bs[best_perm[s]]);
                    bsel[gid][s] = bs[best_perm[s]];
                    fsel[gid][s] = fs[best_perm[s]];
                }
            }
            // ones rows: the least used bank group of the load that reads them
            auto one_code = [&](const std::vector<int>& rows) {
                int c[4] = {0, 0, 0, 0};
                std::vector<int> seen;
                for (int r : rows)
                    if (r != ONE && std::find(seen.begin(), seen.end(), r) == seen.end()) { seen.push_back(r); c[cls(r)]++; }
                return kRowOne + 2 * (int)(std::min_element(c, c + 4) - c);
            };
            const int a_one = one_code(std::vector<int>(asel.begin(), asel.end()));
            for (int s = 0; s < 4; s++) {
                const int b_one = one_code(slot_rows[s]);
                for (int gid = 0; gid < 8; gid++) {
                    MRow& o = out[(size_t)mt * 128 + (s >> 1) * 64 + w * 16 + gid + 8 * (s & 1)];
                    o.a = asel[gid] == ONE ? a_one : asel[gid];
                    o.b = bsel[gid][s] == ONE ? b_one : bsel[gid][s];
                    const int f = fsel[gid][s];
                    if (f < 0) continue;
                    o.f = f;
                    if (f == 0) continue;
                    if (f <= D) { o.i = f - 1; continue; }
                    const Item* it = nullptr;
                    for (const Item& x : items) if (x.f == f) it = &x;
                    o.i = it->i;
                    o.j = it->j;
                }
            }
        }
    }
    return out;
}

}  // namespace gmm
