// Host build of the two-class SWAR word (skywalking-banyandb_b200/csrc/lane_decode.cuh: swar_word2) with the switch to the
// three-class swar_word that the express lane applies per chunk (scan_kernels.cu: swar_chunk_sum): whole pages emulated lane
// by lane against the plain definition of the page sum.
// Built and run by tests/test_lane_switch_native.py with g++ (the CUDA toolkit headers only provide uint4).
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <random>
#include <utility>
#include <vector>

#include "lane_decode.cuh"

using namespace bydb;

static int32_t zz(uint32_t u) { return static_cast<int32_t>(u >> 1) ^ -static_cast<int32_t>(u & 1u); }

// ---- the two-class SWAR word (swar_word2) with the switch rule of swar_chunk_sum (scan_kernels.cu): a page starts on the
// two-class word; a chunk whose lanes raise its flag is decoded again from the same carry word with swar_word, which takes
// the rest of the page, where a raised flag (a varint of 4+ bytes) bails the page out.  The page holds 1-2 byte varints
// with longer ones at chosen window offsets (`longs`: start offset, length), so that lane (64 B) and chunk (2 KB)
// boundaries fall before any of their bytes.  Checked against the plain definition, and that the switch happens exactly in
// the chunk that holds the first long varint's second byte.
static bool swar_switch_page_check(std::mt19937_64 &rng, uint32_t pstart, uint32_t body_len, const std::vector<std::pair<uint32_t, int>> &longs) {
    std::vector<int64_t> d;
    std::vector<uint8_t> win(pstart);
    for (auto &x : win) x = static_cast<uint8_t>(rng());
    auto push = [&](int L) {
        uint32_t u = static_cast<uint32_t>(rng()) & ((1u << (7 * L)) - 1u);
        if (L > 1 && (u >> (7 * (L - 1))) == 0) u |= 1u << (7 * (L - 1));
        if (rng() % 7 == 0) u &= ~0x3f80u;  // zero middle payload bytes (0x80 continuation bytes)
        if (L > 1 && (u >> (7 * (L - 1))) == 0) u |= 1u << (7 * (L - 1));
        d.push_back(zz(u));
        for (int k = 0; k < L; ++k) win.push_back(static_cast<uint8_t>(((u >> (7 * k)) & 0x7f) | (k < L - 1 ? 0x80 : 0)));
    };
    size_t next = 0;
    int max_len = 2;
    int64_t first_long = -1;
    while (win.size() < pstart + body_len || next < longs.size()) {
        const uint32_t pos = static_cast<uint32_t>(win.size());
        if (next < longs.size() && longs[next].first == pos) {
            push(longs[next].second);
            max_len = longs[next].second > max_len ? longs[next].second : max_len;
            if (first_long < 0) first_long = pos;
            ++next;
        } else if (next < longs.size() && longs[next].first < pos) {
            ++next;  // overlaps the previous long varint: dropped
        } else {
            push(next < longs.size() && longs[next].first - pos == 1 ? 1 : 1 + static_cast<int>(rng() % 2));
        }
    }
    const int n_values = static_cast<int>(d.size());
    const uint32_t pend = static_cast<uint32_t>(win.size());
    while (win.size() % 16) win.push_back(static_cast<uint8_t>(rng()));
    const uint32_t total = static_cast<uint32_t>(win.size());
    win.resize(win.size() + 2048, 0xAB);
    const int64_t n = n_values + 1;
    int64_t want = 0, pre = 0;
    for (int j = 0; j < n_values; ++j) {
        pre += d[j];
        want += pre;
    }
    int64_t S = 0;
    uint32_t tb = 0, carry_w = 0, redone = 0;
    int64_t switch_chunk = -1;
    bool three = false, bailed = false;
    const uint32_t nchunks = (total + 2047) / 2048;
    for (uint32_t c = 0; c < nchunks && !bailed; ++c) {
        const bool interior = c * 2048 >= pstart && (c + 1) * 2048 <= pend;
        uint32_t nl[32], lastw[32];
        int32_t T[32], Rp[32];
        auto run = [&](bool three_class) {
            uint32_t flag = 0;
            for (int lane = 0; lane < 32; ++lane) {
                const uint32_t o = c * 2048 + lane * 64;
                uint32_t w[16];
                for (int k = 0; k < 16; ++k) {
                    w[k] = 0;
                    if (o + 4 * k < total) memcpy(&w[k], &win[o + 4 * k], 4);
                }
                int lo_i = static_cast<int>(pstart) - static_cast<int>(o), hi_i = static_cast<int>(pend) - static_cast<int>(o);
                lo_i = lo_i < 0 ? 0 : (lo_i > 64 ? 64 : lo_i);
                hi_i = hi_i < 0 ? 0 : (hi_i > 64 ? 64 : hi_i);
                const uint64_t valid = (hi_i >= 64 ? ~0ull : ((1ull << hi_i) - 1ull)) & ~(lo_i >= 64 ? ~0ull : ((1ull << lo_i) - 1ull));
                SwarLane sl;
                swar_begin(sl, lane == 0 ? carry_w : lastw[lane - 1]);
                for (int k = 0; k < 16; ++k) {
                    const uint32_t vm = expand4(static_cast<uint32_t>(valid >> (4 * k)));
                    if (three_class) {
                        if (interior) swar_word<false>(sl, w[k], 0xffffffffu);
                        else swar_word<true>(sl, w[k], vm);
                    } else {
                        if (interior) swar_word2<false>(sl, w[k], 0xffffffffu);
                        else swar_word2<true>(sl, w[k], vm);
                    }
                }
                lastw[lane] = sl.prev_w;
                nl[lane] = swar_end(sl, T[lane], Rp[lane]);
                flag |= sl.wide & 0x80808080u;
            }
            return flag != 0;
        };
        bool flag = run(three);
        if (!three && flag) {
            three = true;
            ++redone;
            switch_chunk = c;
            flag = run(true);
        }
        if (flag) {
            bailed = true;
            break;
        }
        carry_w = lastw[31];
        uint32_t lb = 0;
        for (int lane = 0; lane < 32; ++lane) {
            const int64_t A = (n - 1) - static_cast<int64_t>(tb) - static_cast<int64_t>(lb);
            S += (A + 1) * static_cast<int64_t>(T[lane]) - static_cast<int64_t>(Rp[lane]);
            lb += nl[lane];
        }
        tb += lb;
    }
    const int64_t want_switch = first_long < 0 ? -1 : (first_long + 1) / 2048;
    if (switch_chunk != want_switch || redone > 1 || bailed != (max_len > 3)) {
        std::printf("FAIL swar switch: pstart=%u pend=%u first long varint at %lld: switched in chunk %lld (want %lld), bailed=%d max_len=%d\n", pstart, pend,
                    static_cast<long long>(first_long), static_cast<long long>(switch_chunk), static_cast<long long>(want_switch), bailed, max_len);
        return false;
    }
    if (!bailed && (tb != static_cast<uint32_t>(n_values) || S != want)) {
        std::printf("FAIL swar switch page: n_values=%d pstart=%u first long varint at %lld terminators=%u S=%lld want=%lld\n", n_values, pstart,
                    static_cast<long long>(first_long), tb, static_cast<long long>(S), static_cast<long long>(want));
        return false;
    }
    return true;
}

int main() {
    std::mt19937_64 rng(20261015);
    long pages = 0;
    for (int it = 0; it < 4000; ++it) {
        const uint32_t pstart = static_cast<uint32_t>(rng() % 16), len = 1 + static_cast<uint32_t>(rng() % 12000), end = pstart + len;
        auto before = [&](uint32_t B) { return B - static_cast<uint32_t>(rng() % 4); };  // the boundary falls before byte 0, 1 or 2 of the varint, or just after it
        auto lane_edge = [&] { return 64u * (1u + static_cast<uint32_t>(rng() % (end / 64 + 1))); };
        auto chunk_edge = [&] { return 2048u * (1u + static_cast<uint32_t>(rng() % (end / 2048 + 1))); };
        std::vector<std::pair<uint32_t, int>> longs;
        switch (it % 8) {
        case 0: break;                                                                   // 1-2 byte varints only: never switches
        case 1: longs.push_back({before(lane_edge()), 3}); break;                        // across a lane edge
        case 2: longs.push_back({before(chunk_edge()), 3}); break;                       // across a chunk edge
        case 3: longs.push_back({pstart + (rng() % 2 ? 0u : static_cast<uint32_t>(rng() % 64)), 3}); break;  // first chunk
        case 4: longs.push_back({end + static_cast<uint32_t>(rng() % 3), 3}); break;     // the page's last varint
        case 5: {                                                                        // several, in different chunks
            for (int k = 0; k < 6; ++k) longs.push_back({pstart + static_cast<uint32_t>(rng() % len), 3});
            break;
        }
        case 6: {                                                                        // a 4-byte varint after the switch
            const uint32_t a = before(rng() % 2 ? lane_edge() : chunk_edge());
            longs.push_back({a, 3});
            longs.push_back({a + 3 + static_cast<uint32_t>(rng() % 2 ? rng() % 8 : rng() % 5000), 4});
            break;
        }
        default: longs.push_back({before(rng() % 2 ? lane_edge() : chunk_edge()), 4}); break;  // a 4-byte varint raises both flags
        }
        for (auto &l : longs) l.first = l.first < pstart ? pstart : l.first;
        std::sort(longs.begin(), longs.end());
        if (!swar_switch_page_check(rng, pstart, len, longs)) return 1;
        ++pages;
    }
    std::printf("OK %ld pages\n", pages);
    return 0;
}
