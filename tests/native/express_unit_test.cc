// Host build of the express lane's page sum (skywalking-banyandb_b200/csrc/scan_kernels.cu: scan_sum_express_kernel with
// express_zero_edges / express_unit / express_half) over the lane words of lane_decode.cuh: whole pages emulated with the kernel's
// geometry -- one 4 KB stage is one unit of two 2 KB halves, a 64-byte window per lane in each half, the unmasked word on every
// unit with the bytes outside the body zeroed, one packed scan of both halves' terminator counts, tb started at minus the zeros
// in front of the body, the two-class word carrying its rank base, and the redo of a flagged unit with the three-class word --
// against a byte-at-a-time page sum.
// Built and run by tests/test_express_unit_native.py with g++ (the CUDA toolkit headers only provide uint4).
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <random>
#include <utility>
#include <vector>

#include "lane_decode.cuh"

using namespace bydb;

constexpr uint32_t kUnit = 4096, kHalf = 2048, kWin = 64;

static int32_t zz(uint32_t u) { return static_cast<int32_t>(u >> 1) ^ -static_cast<int32_t>(u & 1u); }

struct Page {
    std::vector<uint8_t> win;  // 16-aligned window: garbage [0, pstart), body [pstart, pend), garbage up to total
    uint32_t pstart = 0, pend = 0, total = 0;
    int64_t want = 0;          // sum over rows of (value - first)
    uint32_t n_values = 0;     // varints in the body = count - 1
    int max_len = 0;
    int64_t first_long = -1;   // window offset of the first varint of 3+ bytes
};

struct Result {
    bool good;
    int64_t S;
    int64_t switch_unit;  // unit where the two-class flag was raised (-1: never)
};

// the kernel's per-page loop; `stale`: the byte an unfilled stage position holds
static Result express_page(const Page &pg, uint32_t count, uint8_t stale) {
    const uint32_t nst = (pg.total + kUnit - 1) / kUnit;
    std::vector<uint8_t> stage(kUnit);
    int64_t S = 0;
    int32_t tb = -static_cast<int32_t>(pg.pstart);
    uint32_t carry_w = 0;
    bool three = false, good = true;
    int64_t switch_unit = -1;
    for (uint32_t j = 0; j < nst && good; ++j) {
        // the TMA copy of this stage: min(4 KB, total - off) bytes; the rest of the stage keeps what an earlier copy left
        std::fill(stage.begin(), stage.end(), stale);
        const uint32_t off = j * kUnit, bytes = std::min(kUnit, pg.total - off);
        memcpy(stage.data(), pg.win.data() + off, bytes);
        // express_zero_edges: the bytes of the unit in front of the body and behind it (the next column's, stale ones) made zeros
        if (j == 0 || (j + 1) * kUnit > pg.pend) {
            for (uint32_t i = 0; i < kUnit; ++i)
                if (off + i < pg.pstart || off + i >= pg.pend) stage[i] = 0;
        }
        auto word_at = [&](uint32_t o) {
            uint32_t w;
            memcpy(&w, stage.data() + o, 4);
            return w;
        };
        uint32_t la[32], lb[32];
        for (int lane = 0; lane < 32; ++lane) {
            la[lane] = word_at(lane * kWin + kWin - 4);
            lb[lane] = word_at(kHalf + lane * kWin + kWin - 4);
        }
        int32_t Ta[32], Ra[32], Tb[32], Rb[32];
        uint32_t n[32];
        auto run = [&](int classes) {
            uint32_t flag = 0;
            for (int lane = 0; lane < 32; ++lane) {
                const uint32_t xa = la[(lane + 31) & 31], xb = lb[(lane + 31) & 31];
                const uint32_t pw[2] = {lane == 0 ? carry_w : xa, lane == 0 ? xa : xb};
                uint32_t nh[2];
                for (int h = 0; h < 2; ++h) {
                    SwarLane sl;
                    swar_begin(sl, pw[h]);
                    for (int q = 0; q < 4; ++q) {
                        uint32_t w[4];
                        for (int k = 0; k < 4; ++k) w[k] = word_at(h * kHalf + lane * kWin + 16 * q + 4 * k);
                        for (int k = 0; k < 4; ++k) {
                            if (classes == 2) swar_word2<false>(sl, w[k], 0u);
                            else swar_word<false>(sl, w[k], 0u);
                        }
                    }
                    flag |= sl.wide & 0x80808080u;
                    nh[h] = h == 0 ? swar_end(sl, Ta[lane], Ra[lane]) : swar_end(sl, Tb[lane], Rb[lane]);
                    if (nh[h] > kWin) std::printf("FAIL: %u terminators in a 64-byte window\n", nh[h]);
                }
                n[lane] = nh[0] | (nh[1] << 16);
            }
            return flag != 0;
        };
        bool wide = false;
        if (!three) {
            wide = run(2);
            three = wide;
            if (three) switch_unit = j;
        }
        if (three) wide = run(3);
        carry_w = lb[31];
        if (wide) {
            good = false;
            break;
        }
        uint32_t incl[32], acc = 0;
        for (int lane = 0; lane < 32; ++lane) incl[lane] = acc += n[lane];
        const uint32_t tot = incl[31];
        for (int lane = 0; lane < 32; ++lane) {
            const uint32_t ex = incl[lane] - n[lane];
            const int32_t Aa = static_cast<int32_t>(count) - tb - static_cast<int32_t>(ex & 0xffffu);
            const int32_t Ab = Aa - static_cast<int32_t>(tot & 0xffffu) + static_cast<int32_t>(ex & 0xffffu) - static_cast<int32_t>(ex >> 16);
            S += static_cast<int64_t>(Aa) * Ta[lane] + static_cast<int64_t>(Ab) * Tb[lane] - Ra[lane] - Rb[lane];
        }
        tb += static_cast<int32_t>((tot & 0xffffu) + (tot >> 16));
    }
    const int32_t zeros_after = static_cast<int32_t>(nst * kUnit - pg.pend);
    const uint8_t last_byte = pg.win[pg.pend - 1];
    good = good && tb - zeros_after + 1 == static_cast<int32_t>(count) && last_byte < 0x80u;
    return {good, S, switch_unit};
}

// A body of `len` bytes (the last varint may run past it) of 1-2 byte varints (`one`: 1-byte only), with the varints of
// `longs` (body offset, length) placed where they fall on a varint start.
static Page make_page(std::mt19937_64 &rng, uint32_t pstart, uint32_t len, bool one, std::vector<std::pair<uint32_t, int>> longs) {
    Page pg;
    pg.pstart = pstart;
    for (uint32_t i = 0; i < pstart; ++i) pg.win.push_back(static_cast<uint8_t>(rng() | 0x80));  // header bytes: continuations at worst
    std::vector<int64_t> d;
    auto push = [&](int L) {
        uint32_t u = static_cast<uint32_t>(rng()) & ((1u << (7 * L)) - 1u);
        if (rng() % 5 == 0) u &= ~0x3f80u;  // zero middle payload bytes (0x80 continuation bytes)
        if (L > 1 && (u >> (7 * (L - 1))) == 0) u |= 1u << (7 * (L - 1));
        d.push_back(zz(u));
        for (int k = 0; k < L; ++k) pg.win.push_back(static_cast<uint8_t>(((u >> (7 * k)) & 0x7f) | (k < L - 1 ? 0x80 : 0)));
        pg.max_len = std::max(pg.max_len, L);
    };
    std::sort(longs.begin(), longs.end());
    size_t next = 0;
    while (pg.win.size() < pstart + len) {
        const uint32_t pos = static_cast<uint32_t>(pg.win.size()) - pstart;
        while (next < longs.size() && longs[next].first < pos) ++next;  // overlaps the previous varint: dropped
        if (next < longs.size() && longs[next].first == pos) {
            if (pg.first_long < 0) pg.first_long = pstart + pos;
            push(longs[next++].second);
        } else {
            const uint32_t room = next < longs.size() ? longs[next].first - pos : 2;
            push(one || room == 1 ? 1 : 1 + static_cast<int>(rng() % 2));
        }
    }
    pg.pend = static_cast<uint32_t>(pg.win.size());
    pg.n_values = static_cast<uint32_t>(d.size());
    while (pg.win.size() % 16) pg.win.push_back(static_cast<uint8_t>(rng() | 0x80));  // the next column's bytes
    pg.total = static_cast<uint32_t>(pg.win.size());
    int64_t pre = 0;
    for (int64_t x : d) {
        pre += x;
        pg.want += pre;
    }
    return pg;
}

static bool check(std::mt19937_64 &rng, uint32_t pstart, uint32_t len, bool one, const std::vector<std::pair<uint32_t, int>> &longs, const char *what) {
    const Page pg = make_page(rng, pstart, len, one, longs);
    const uint32_t count = pg.n_values + 1;
    for (uint8_t stale : {static_cast<uint8_t>(0xff), static_cast<uint8_t>(0x00)}) {
        const Result r = express_page(pg, count, stale);
        const bool want_bail = pg.max_len > 3;
        const int64_t want_switch = pg.first_long < 0 ? -1 : (pg.first_long + 1) / kUnit;  // the unit of the long varint's second byte
        if (r.good == want_bail || r.switch_unit != want_switch || (r.good && r.S != pg.want)) {
            std::printf("FAIL %s: pstart=%u pend=%u total=%u stale=0x%02x max_len=%d first_long=%lld good=%d switch_unit=%lld (want %lld) S=%lld want=%lld\n",
                        what, pstart, pg.pend, pg.total, stale, pg.max_len, static_cast<long long>(pg.first_long), r.good,
                        static_cast<long long>(r.switch_unit), static_cast<long long>(want_switch), static_cast<long long>(r.S),
                        static_cast<long long>(pg.want));
            return false;
        }
        // a count that does not match the body must fail the check
        if (!want_bail && express_page(pg, count + 1, stale).good) {
            std::printf("FAIL %s: pstart=%u pend=%u accepted a wrong row count\n", what, pstart, pg.pend);
            return false;
        }
    }
    return true;
}

int main() {
    std::mt19937_64 rng(20261015);
    long pages = 0;
    // body lengths at +-1 around the 16-byte piece, 64-byte window, 2 KB half and 4 KB unit edges (and a few multiples)
    std::vector<uint32_t> lens;
    for (uint32_t e : {16u, 64u, 2048u, 4096u, 3u * 16u, 5u * 64u, 3u * 2048u, 2u * 4096u, 4u * 4096u})
        for (int dl = -1; dl <= 1; ++dl) lens.push_back(e + dl);
    lens.push_back(1);
    lens.push_back(2);
    lens.push_back(15800);  // about a bench page
    for (uint32_t pstart = 0; pstart < 16; ++pstart) {
        for (uint32_t len : lens) {
            if (!check(rng, pstart, len, false, {}, "1-2 byte varints")) return 1;
            if (!check(rng, pstart, len, true, {}, "1-byte varints (64 terminators per window)")) return 1;
            ++pages;
            // a 3-byte varint starting just before, on and after every half and unit edge of the body, and in the first window
            for (uint32_t edge = 0; edge <= len + kHalf; edge += kHalf) {
                for (int at = -3; at <= 1; ++at) {
                    const int64_t w = static_cast<int64_t>(edge) + at - pstart;  // window offset -> body offset
                    if (w < 0 || w >= len) continue;
                    if (!check(rng, pstart, len, false, {{static_cast<uint32_t>(w), 3}}, "3-byte varint at a half / unit edge")) return 1;
                    ++pages;
                }
            }
            if (len > 8) {
                // 3-byte varints at random places, the last one possibly the body's last varint
                std::vector<std::pair<uint32_t, int>> longs;
                for (int k = 0; k < 4; ++k) longs.push_back({static_cast<uint32_t>(rng() % len), 3});
                if (!check(rng, pstart, len, false, longs, "3-byte varints")) return 1;
                // a 4-byte varint after the switch (same unit or a later one), and a 4-byte varint alone
                const uint32_t a = static_cast<uint32_t>(rng() % (len / 2 + 1));
                const uint32_t b = std::min(len - 1, a + 3 + static_cast<uint32_t>(rng() % 2 ? rng() % 8 : rng() % 5000));
                if (b > a + 2 && !check(rng, pstart, len, false, {{a, 3}, {b, 4}}, "4-byte varint after the switch")) return 1;
                if (!check(rng, pstart, len, false, {{static_cast<uint32_t>(rng() % len), 4}}, "4-byte varint")) return 1;
                pages += 3;
            }
        }
    }
    std::printf("OK %ld pages\n", pages);
    return 0;
}
