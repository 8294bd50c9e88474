// Host build of the per-lane fast decoders (skywalking-banyandb_b200/csrc/lane_decode.cuh) against a byte-at-a-time reference:
//   * fast_lane_decode<true>   interior chunk (all 32 bytes valid), every kNeed variant
//   * fast_lane_decode<false>  chunk with bytes outside the page (first / last chunk), random valid windows
//   * swar_word / swar_end     the SWAR sum decoder, a whole page emulated lane by lane against the plain definition
//   * head_delta               the cross-lane / cross-half correction identity
// Built and run by tests/test_lane_decode_native.py with g++ (the CUDA toolkit headers only provide uint4).
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

#include "lane_decode.cuh"

using namespace bydb;

struct Ref {
    uint32_t accv = 0, sh = 0;
    int32_t P = 0, sumP = 0, minP = INT32_MAX, maxP = INT32_MIN;
};
static int32_t zz(uint32_t u) { return static_cast<int32_t>(u >> 1) ^ -static_cast<int32_t>(u & 1u); }

// the semantics the kernel documents: only valid bytes exist; invalid bytes restart the varint state
static Ref reference(const uint8_t *b, uint32_t valid, uint32_t aw) {
    Ref r;
    for (int i = 0; i < 32; ++i) {
        if (!((valid >> i) & 1u)) {
            r.accv = 0;
            r.sh = 0;
            continue;
        }
        r.accv |= static_cast<uint32_t>(b[i] & 0x7f) << r.sh;
        r.sh += 7;
        if (b[i] < 0x80) {
            r.P += zz(r.accv);
            if (aw & 1u) {
                r.sumP += r.P;
                r.minP = r.P < r.minP ? r.P : r.minP;
                r.maxP = r.P > r.maxP ? r.P : r.maxP;
            }
            aw >>= 1;
            r.accv = 0;
            r.sh = 0;
        }
    }
    return r;
}

template <bool kFull, int kNeed>
static bool check(const uint8_t *b, uint32_t valid, uint32_t aw) {
    uint4 wa, wb;
    uint32_t w[8];
    for (int k = 0; k < 8; ++k) w[k] = b[4 * k] | (b[4 * k + 1] << 8) | (b[4 * k + 2] << 16) | (static_cast<uint32_t>(b[4 * k + 3]) << 24);
    wa = {w[0], w[1], w[2], w[3]};
    wb = {w[4], w[5], w[6], w[7]};
    uint32_t msb = 0;
    for (int k = 0; k < 8; ++k) msb |= msb4(w[k]) << (4 * k);
    const uint32_t term = valid & ~msb;
    uint32_t accv = 0, sh = 0;
    int32_t P = 0, sumP = 0, minP = INT32_MAX, maxP = INT32_MIN;
    fast_lane_decode<kFull, kNeed>(wa, wb, valid, term, aw, accv, sh, P, sumP, minP, maxP);
    const Ref r = reference(b, valid, aw);
    bool ok = accv == r.accv && sh == r.sh && P == r.P;
    if (kNeed & kNeedSum) ok = ok && sumP == r.sumP;
    if (kNeed & kNeedMinMax) ok = ok && minP == r.minP && maxP == r.maxP;
    if (!ok)
        std::printf("FAIL full=%d need=%d valid=%08x aw=%08x: got (%u,%u,%d,%d,%d,%d) want (%u,%u,%d,%d,%d,%d)\n", kFull, kNeed, valid, aw,
                    accv, sh, P, sumP, minP, maxP, r.accv, r.sh, r.P, r.sumP, r.minP, r.maxP);
    return ok;
}

// ---- SWAR sum decoder (swar_begin / swar_word / swar_end): a whole page emulated lane by lane exactly like the kernel
// walks it (2 KB chunks of 32 lanes x 64 bytes, 16-byte aligned window around the page, masked first / last chunk, the
// previous lane's last word handed on, per-chunk exclusive scan of the lanes' terminator counts), against the plain
// definition  sum over rows of (first + prefix of the deltas).
static bool swar_page_check(std::mt19937_64 &rng, int n_values, int max_len) {
    std::vector<int64_t> d;
    std::vector<uint8_t> body;
    const uint32_t pstart = static_cast<uint32_t>(rng() % 16);
    std::vector<uint8_t> win(pstart);
    for (auto &x : win) x = static_cast<uint8_t>(rng());  // bytes of a neighbouring page in front of this one
    for (int i = 0; i < n_values; ++i) {
        const int L = 1 + static_cast<int>(rng() % max_len);
        uint32_t u = static_cast<uint32_t>(rng()) & ((1u << (7 * L)) - 1u);
        if (L > 1 && (u >> (7 * (L - 1))) == 0) u |= 1u << (7 * (L - 1));
        if (rng() % 7 == 0) u &= ~0x3f80u;  // zero middle payload bytes (0x80 continuation bytes)
        if (L > 1 && (u >> (7 * (L - 1))) == 0) u |= 1u << (7 * (L - 1));
        d.push_back(zz(u));
        for (int k = 0; k < L; ++k) win.push_back(static_cast<uint8_t>(((u >> (7 * k)) & 0x7f) | (k < L - 1 ? 0x80 : 0)));
    }
    const uint32_t pend = static_cast<uint32_t>(win.size());
    while (win.size() % 16) win.push_back(static_cast<uint8_t>(rng()));
    const uint32_t total = static_cast<uint32_t>(win.size());
    win.resize(win.size() + 2048, 0xAB);  // reads past `total` never happen in the kernel; keep the emulation honest with junk
    // reference
    const int64_t n = n_values + 1;
    int64_t want = 0, pre = 0;
    for (int j = 0; j < n_values; ++j) {
        pre += d[j];
        want += pre;
    }
    // emulation
    int64_t S = 0;
    uint32_t tb = 0, carry_w = 0, wide = 0;
    const uint32_t nchunks = (total + 2047) / 2048;
    for (uint32_t c = 0; c < nchunks; ++c) {
        const bool interior = c * 2048 >= pstart && (c + 1) * 2048 <= pend;
        uint32_t nl[32], lastw[32];
        int32_t T[32], Rp[32];
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
            // previous lane's last word: masked like that lane saw it
            uint32_t pw = lane == 0 ? carry_w : lastw[lane - 1];
            SwarLane sl;
            swar_begin(sl, pw);
            for (int k = 0; k < 16; ++k) {
                if (interior) swar_word<false>(sl, w[k], 0xffffffffu);
                else swar_word<true>(sl, w[k], expand4(static_cast<uint32_t>(valid >> (4 * k))));
            }
            lastw[lane] = sl.prev_w;
            nl[lane] = swar_end(sl, T[lane], Rp[lane]);
            wide |= sl.wide;
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
    const bool is_wide = (wide & 0x80808080u) != 0;
    if (max_len > 3) {
        bool has_wide = false;
        // (only checks that a 4+ byte varint is flagged)
        uint32_t run = 0;
        for (uint32_t i = pstart; i < pend; ++i) {
            run = (win[i] & 0x80) ? run + 1 : 0;
            if (run >= 3) has_wide = true;
        }
        if (has_wide != is_wide) {
            std::printf("FAIL swar wide flag: has=%d flagged=%d\n", has_wide, is_wide);
            return false;
        }
        if (has_wide) return true;
    } else if (is_wide) {
        std::printf("FAIL swar: narrow page flagged wide\n");
        return false;
    }
    if (tb != static_cast<uint32_t>(n_values) || S != want) {
        std::printf("FAIL swar page: n_values=%d pstart=%u terminators=%u S=%lld want=%lld\n", n_values, pstart, tb, static_cast<long long>(S),
                    static_cast<long long>(want));
        return false;
    }
    return true;
}

// ---- SWAR sum under a row mask (swar_masked_*): a page emulated the way delta_page_sum_masked walks it -- first the lanes' terminator
// counts (row offsets), then the words with the rank taken over ACTIVE terminators -- against the plain masked sum.
static bool swar_masked_page_check(std::mt19937_64 &rng, int n_values, int density_pct) {
    std::vector<int64_t> d;
    const uint32_t pstart = static_cast<uint32_t>(rng() % 16);
    std::vector<uint8_t> win(pstart);
    for (auto &x : win) x = static_cast<uint8_t>(rng());
    for (int i = 0; i < n_values; ++i) {
        const int L = 1 + static_cast<int>(rng() % 3);
        uint32_t u = static_cast<uint32_t>(rng()) & ((1u << (7 * L)) - 1u);
        if (L > 1 && (u >> (7 * (L - 1))) == 0) u |= 1u << (7 * (L - 1));
        if (rng() % 7 == 0) u &= ~0x3f80u;
        if (L > 1 && (u >> (7 * (L - 1))) == 0) u |= 1u << (7 * (L - 1));
        d.push_back(zz(u));
        for (int k = 0; k < L; ++k) win.push_back(static_cast<uint8_t>(((u >> (7 * k)) & 0x7f) | (k < L - 1 ? 0x80 : 0)));
    }
    const uint32_t pend = static_cast<uint32_t>(win.size());
    while (win.size() % 16) win.push_back(static_cast<uint8_t>(rng()));
    const uint32_t total = static_cast<uint32_t>(win.size());
    win.resize(win.size() + 2048, 0xAB);
    const int64_t first = static_cast<int64_t>(rng() % 2000001) - 1000000;
    std::vector<uint8_t> act(n_values + 1 + 128, 0);
    for (size_t r = 0; r < static_cast<size_t>(n_values) + 1;) {
        const size_t run = 1 + rng() % 40;
        const bool on = static_cast<int>(rng() % 100) < density_pct;
        for (size_t k = 0; k < run && r < static_cast<size_t>(n_values) + 1; ++k) act[r++] = on;
    }
    int64_t want = 0, A_total = 0, v = first;
    for (int r = 0; r <= n_values; ++r) {
        if (r > 0) v += d[r - 1];
        if (act[r]) {
            want += v;
            A_total++;
        }
    }
    int64_t S = 0;
    uint32_t row_base = 1, atb = 0, carry_w = 0;
    const uint32_t nchunks = (total + 2047) / 2048;
    for (uint32_t c = 0; c < nchunks; ++c) {
        const bool interior = c * 2048 >= pstart && (c + 1) * 2048 <= pend;
        uint32_t lastw[32], nall[32], nact[32];
        int32_t T[32], Rp[32];
        uint64_t valid[32];
        uint32_t w[32][16];
        for (int lane = 0; lane < 32; ++lane) {
            const uint32_t o = c * 2048 + lane * 64;
            for (int k = 0; k < 16; ++k) {
                w[lane][k] = 0;
                if (o + 4 * k < total) memcpy(&w[lane][k], &win[o + 4 * k], 4);
            }
            int lo_i = static_cast<int>(pstart) - static_cast<int>(o), hi_i = static_cast<int>(pend) - static_cast<int>(o);
            lo_i = lo_i < 0 ? 0 : (lo_i > 64 ? 64 : lo_i);
            hi_i = hi_i < 0 ? 0 : (hi_i > 64 ? 64 : hi_i);
            valid[lane] = (hi_i >= 64 ? ~0ull : ((1ull << hi_i) - 1ull)) & ~(lo_i >= 64 ? ~0ull : ((1ull << lo_i) - 1ull));
            nall[lane] = 0;
            for (int k = 0; k < 16; ++k) nall[lane] += count_terminators(w[lane][k], interior ? 0xffffffffu : expand4(static_cast<uint32_t>(valid[lane] >> (4 * k))));
        }
        uint32_t lb = 0;
        for (int lane = 0; lane < 32; ++lane) {
            const uint32_t row0 = row_base + lb;
            uint64_t aw = 0;
            for (uint32_t i = 0; i < nall[lane] && i < 64; ++i) aw |= static_cast<uint64_t>(act[row0 + i]) << i;
            SwarMasked sl;
            swar_masked_begin(sl, lane == 0 ? carry_w : lastw[lane - 1], static_cast<uint32_t>(aw), static_cast<uint32_t>(aw >> 32));
            for (int k = 0; k < 16; ++k) {
                if (interior) swar_masked_word<false>(sl, w[lane][k], 0xffffffffu);
                else swar_masked_word<true>(sl, w[lane][k], expand4(static_cast<uint32_t>(valid[lane] >> (4 * k))));
            }
            lastw[lane] = sl.prev_w;
            nact[lane] = swar_masked_end(sl, T[lane], Rp[lane]);
            if ((sl.wide & 0x80808080u) != 0) {
                std::printf("FAIL masked swar: narrow page flagged wide\n");
                return false;
            }
            if (nact[lane] != static_cast<uint32_t>(__builtin_popcountll(aw))) {
                std::printf("FAIL masked swar: active terminators %u vs %d (chunk %u lane %d)\n", nact[lane], __builtin_popcountll(aw), c, lane);
                return false;
            }
            lb += nall[lane];
        }
        carry_w = lastw[31];
        uint32_t alb = 0;
        for (int lane = 0; lane < 32; ++lane) {
            const int64_t A1a = (A_total - act[0]) - static_cast<int64_t>(atb) - static_cast<int64_t>(alb) + 1;
            S += A1a * static_cast<int64_t>(T[lane]) - static_cast<int64_t>(Rp[lane]);
            alb += nact[lane];
        }
        atb += alb;
        row_base += lb;
    }
    const int64_t got = A_total * first + S;
    if (row_base != static_cast<uint32_t>(n_values) + 1 || got != want || static_cast<int64_t>(atb) + act[0] != A_total) {
        std::printf("FAIL masked swar page: n_values=%d pstart=%u rows=%u got=%lld want=%lld active=%u/%lld\n", n_values, pstart, row_base,
                    static_cast<long long>(got), static_cast<long long>(want), atb + act[0], static_cast<long long>(A_total));
        return false;
    }
    return true;
}

int main() {
    std::mt19937_64 rng(20260922);
    long n = 0;
    for (int it = 0; it < 200000; ++it) {
        // a stream of narrow (1..3 byte) varints, window cut at a random offset
        std::vector<uint8_t> s;
        while (s.size() < 48) {
            const int L = 1 + static_cast<int>(rng() % 3);
            uint32_t u = static_cast<uint32_t>(rng()) & ((1u << (7 * L)) - 1u);
            if (L > 1 && (u >> (7 * (L - 1))) == 0) u |= 1u << (7 * (L - 1));  // canonical length
            for (int k = 0; k < L; ++k) s.push_back(static_cast<uint8_t>(((u >> (7 * k)) & 0x7f) | (k < L - 1 ? 0x80 : 0)));
        }
        const uint8_t *b = s.data() + rng() % 4;
        const uint32_t aw = (rng() % 4 == 0) ? 0xffffffffu : (rng() % 5 == 0 ? 0u : static_cast<uint32_t>(rng()));
        bool ok = check<true, kNeedSum>(b, 0xffffffffu, aw) && check<true, kNeedMinMax>(b, 0xffffffffu, aw) &&
                  check<true, kNeedSum | kNeedMinMax>(b, 0xffffffffu, aw);
        // first / last chunk of a page: a contiguous valid window [lo, hi)
        const uint32_t lo = rng() % 33, hi = lo + rng() % (33 - lo);
        const uint32_t valid = (hi >= 32 ? 0xffffffffu : ((1u << hi) - 1u)) & ~(lo >= 32 ? 0xffffffffu : ((1u << lo) - 1u));
        ok = ok && check<false, kNeedSum>(b, valid, aw) && check<false, kNeedSum | kNeedMinMax>(b, valid, aw);
        if (!ok) return 1;
        n += 8;
    }
    // head_delta: value split between a previous tail (prev_acc, prev_sh) and the first 1..2 bytes of this lane
    for (int it = 0; it < 100000; ++it) {
        const int L = 2 + static_cast<int>(rng() % 2), cut = 1 + static_cast<int>(rng() % (L - 1));
        const uint32_t u = static_cast<uint32_t>(rng()) & ((1u << (7 * L)) - 1u);
        uint8_t bytes[3];
        for (int k = 0; k < L; ++k) bytes[k] = static_cast<uint8_t>(((u >> (7 * k)) & 0x7f) | (k < L - 1 ? 0x80 : 0));
        uint32_t prev_acc = 0;
        for (int k = 0; k < cut; ++k) prev_acc |= static_cast<uint32_t>(bytes[k] & 0x7f) << (7 * k);
        uint32_t w0 = 0, hx = 0;
        for (int k = cut; k < L; ++k) {
            w0 |= static_cast<uint32_t>(bytes[k]) << (8 * (k - cut));
            hx |= static_cast<uint32_t>(bytes[k] & 0x7f) << (7 * (k - cut));
        }
        w0 |= static_cast<uint32_t>(rng()) << (8 * (L - cut));  // whatever follows in the word
        const uint32_t term = 1u << (L - cut - 1);
        if (head_delta(w0, term | (static_cast<uint32_t>(rng()) << (L - cut)), prev_acc, 7u * cut) != zz(u) - zz(hx)) {
            std::printf("FAIL head_delta u=%u L=%d cut=%d\n", u, L, cut);
            return 1;
        }
        (void)term;
    }
    for (int it = 0; it < 3000; ++it) {
        const int nv = it < 50 ? it : 1 + static_cast<int>(rng() % 9000);
        if (!swar_page_check(rng, nv, 3)) return 1;
        if (it % 10 == 0 && !swar_page_check(rng, nv, 4)) return 1;
    }
    for (int it = 0; it < 3000; ++it) {
        const int nv = it < 50 ? it : 1 + static_cast<int>(rng() % 9000);
        if (!swar_masked_page_check(rng, nv, it % 4 == 0 ? 12 : (it % 4 == 1 ? 50 : (it % 4 == 2 ? 100 : 0)))) return 1;
    }
    std::printf("OK %ld lane decodes\n", n);
    return 0;
}
