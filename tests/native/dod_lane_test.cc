// Host build of the fast lane's delta-of-delta page decoder (skywalking-banyandb_b200/csrc/scan_kernels.cu: dod_page_fast with
// fast_chunk_load) over the lane functions of lane_decode.cuh: whole pages emulated with the kernel's geometry -- the first
// difference read alone, the second differences streamed from the byte after it in a 16 B-aligned copy (32 B per lane, 1 KB
// chunks, two chunks per 2 KB TMA stage, a two-stage ring), the byte masks and the wide check of fast_chunk_load, pass 1
// (fast_lane_decode<kNeedSum>: per-lane prefix P and sum of prefixes sumP, then the head fix sumP += dlt * n), the warp scan
// of (n, q, r) with r = rA + rB + nB*qA, pass 2 and the carries to the next chunk -- against a byte-at-a-time decode.  On a
// bail-out the stage accounting of stream_drain is checked: every stage issued has been waited for and the warp's stage
// sequence moves on by exactly the stages issued.
// Built and run by tests/test_dod_lane_native.py with g++ (the CUDA toolkit headers only provide uint4).
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

#include "lane_decode.cuh"

using namespace bydb;

constexpr uint32_t kStageBytes = 2048, kStages = 2;
constexpr uint32_t kChunksPerStage = kStageBytes / kFastChunkBytes;

static uint64_t zz_enc(int64_t v) { return (static_cast<uint64_t>(v) << 1) ^ static_cast<uint64_t>(v >> 63); }
static int64_t zz_dec(uint64_t u) { return static_cast<int64_t>(u >> 1) ^ -static_cast<int64_t>(u & 1); }
static int64_t wadd(int64_t a, int64_t b) { return static_cast<int64_t>(static_cast<uint64_t>(a) + static_cast<uint64_t>(b)); }
static int64_t wmul(uint64_t a, int64_t b) { return static_cast<int64_t>(a * static_cast<uint64_t>(b)); }
static void put_varint(std::vector<uint8_t> &o, int64_t v) {
    uint64_t u = zz_enc(v);
    while (u >= 0x80) {
        o.push_back(static_cast<uint8_t>(u) | 0x80);
        u >>= 7;
    }
    o.push_back(static_cast<uint8_t>(u));
}

struct Page {
    std::vector<uint8_t> body;  // first difference, then the second differences
    uint32_t body_start = 0;    // where body[0] falls in its 16 B-aligned copy
    int64_t first = 0;
    uint32_t count = 0;         // rows: varints + 1
};

// the reference: one varint after the other (delta.go:91-118)
static bool plain_decode(const Page &pg, std::vector<int64_t> &out) {
    out.assign(1, pg.first);
    uint64_t u = 0;
    uint32_t sh = 0, k = 0;
    int64_t d = 0;
    for (uint8_t b : pg.body) {
        u |= static_cast<uint64_t>(b & 0x7f) << sh;
        sh += 7;
        if (b < 0x80) {
            const int64_t x = zz_dec(u);
            d = k == 0 ? x : wadd(d, x);
            out.push_back(wadd(out.back(), d));
            u = 0;
            sh = 0;
            ++k;
        }
    }
    return sh == 0 && out.size() == pg.count;
}

struct Outcome {
    int rc = 2;               // dod_page_fast's return: 0 done, 1 a varint of 4+ bytes (bail-out), 2 corrupt
    int64_t bail_chunk = -1;
    std::vector<int64_t> vals;
    const char *why = "";
};

// one lane's values, decoded from its own bytes plus the previous lane's unfinished tail (pass 2's loop, without the base)
static void lane_values(const uint4 &wa, const uint4 &wb, uint32_t valid, uint32_t term, uint32_t acc, uint32_t sh, std::vector<int32_t> &xs) {
    const uint32_t w[8] = {wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w};
    for (int j = 0; j < 32; ++j) {
        const uint32_t b = (w[j >> 2] >> (8 * (j & 3))) & 0xffu;
        if ((valid >> j) & 1u) {
            acc |= (b & 0x7fu) << sh;
            sh += 7;
        }
        if ((term >> j) & 1u) {
            xs.push_back(static_cast<int32_t>(acc >> 1) ^ -static_cast<int32_t>(acc & 1u));
            acc = 0;
            sh = 0;
        }
    }
}

// A narrow lane's P and sumP stay far inside int32: a lane ends at most 32 varints, each of at most 3 bytes (|x| <= 2^20, the
// wide check admits no longer run), so |P| <= 11 * 2^20 (at most 11 of them can be 3-byte ones in 32 + 2 bytes) and
// |sumP| <= 32 * 11 * 2^20 < 2^29 with the head fix included (|dlt| < 2^21, dlt * n < 2^26).
constexpr int64_t kSumPBound = 32ll * 11 * (1ll << 20) + 32ll * (1ll << 21);

static Outcome dod_page_emulated(const Page &pg, uint8_t garbage) {
    Outcome out;
    if (pg.count < 2) return out;
    // read_varint_seq: the first difference, at most 10 bytes
    uint64_t u = 0;
    uint32_t used = 0;
    for (uint32_t i = 0; i < pg.body.size() && i < 10; ++i) {
        u |= static_cast<uint64_t>(pg.body[i] & 0x7f) << (7 * i);
        if (pg.body[i] < 0x80) {
            used = i + 1;
            break;
        }
    }
    if (used == 0) return out;
    const int64_t d1 = zz_dec(u);
    out.vals = {pg.first, wadd(pg.first, d1)};
    const uint32_t len = static_cast<uint32_t>(pg.body.size()) - used;
    if (len == 0) {
        out.rc = pg.count == 2 ? 0 : 2;
        return out;
    }
    // stream_open: the 16 B-aligned copy of the second differences
    const uint32_t pstart = (pg.body_start + used) & 15u, pend = pstart + len, total = (pend + 15u) & ~15u;
    const uint32_t nstages = (total + kStageBytes - 1) / kStageBytes;
    std::vector<uint8_t> win(total, garbage);
    memcpy(win.data() + pstart, pg.body.data() + used, len);
    for (uint32_t i = 0; i < pstart && i < used; ++i) win[pstart - 1 - i] = pg.body[used - 1 - i];  // the first difference's bytes
    std::vector<int> waited(nstages, 0);
    uint32_t issued = std::min(nstages, kStages);
    const uint32_t nchunks = (total + kFastChunkBytes - 1) / kFastChunkBytes;
    int64_t V0 = wadd(pg.first, d1), D0 = d1;
    uint32_t carry_acc = 0, carry_sh = 0, row_base = 2;
    out.vals.resize(pg.count + 64, 0);
    for (uint32_t c = 0; c < nchunks; ++c) {
        const uint32_t k = c / kChunksPerStage;
        if (c % kChunksPerStage == 0) {
            if (k >= issued) {
                out.why = "waited for a stage never issued";
                return out;
            }
            waited[k] = 1;
        }
        // ---- fast_chunk_load
        uint4 wa[32], wb[32];
        uint32_t valid[32], term[32], cont[32], n[32], lead[32], trail[32];
        bool all_full = true;
        for (int lane = 0; lane < 32; ++lane) {
            const uint32_t o = c * kFastChunkBytes + lane * kFastLaneBytes;
            uint32_t w[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            if (o < total) memcpy(w, win.data() + o, 16);
            if (o + 16 < total) memcpy(w + 4, win.data() + o + 16, 16);
            wa[lane] = make_uint4(w[0], w[1], w[2], w[3]);
            wb[lane] = make_uint4(w[4], w[5], w[6], w[7]);
            int lo_i = static_cast<int>(pstart) - static_cast<int>(o), hi_i = static_cast<int>(pend) - static_cast<int>(o);
            lo_i = std::min(std::max(lo_i, 0), 32);
            hi_i = std::min(std::max(hi_i, 0), 32);
            valid[lane] = low_bits(hi_i) & ~low_bits(lo_i);
            uint32_t msb = 0;
            for (int q = 0; q < 8; ++q) msb |= msb4(w[q]) << (4 * q);
            term[lane] = valid[lane] & ~msb;
            cont[lane] = valid[lane] & msb;
            n[lane] = lane_popc(term[lane]);
            lead[lane] = term[lane] ? static_cast<uint32_t>(lane_ffs(term[lane]) - 1 - lo_i) : static_cast<uint32_t>(hi_i - lo_i);
            trail[lane] = term[lane] ? static_cast<uint32_t>(hi_i - 1 - (31 - lane_clz(term[lane]))) : static_cast<uint32_t>(hi_i - lo_i);
            all_full = all_full && valid[lane] == 0xffffffffu;
        }
        bool wide = false;
        for (int lane = 0; lane < 32; ++lane) {
            const uint32_t trail_prev = lane == 0 ? carry_sh / 7 : trail[lane - 1];
            wide = wide || (cont[lane] & (cont[lane] >> 1) & (cont[lane] >> 2)) != 0 || trail_prev + lead[lane] > 2;
        }
        if (wide) {
            // stream_drain(k): wait for stages k+1 .. issued-1; the warp's sequence moves on by min(nstages, k + kStages)
            const uint32_t seq_next = std::min(nstages, k + kStages);
            for (uint32_t j = k + 1; j < seq_next; ++j) waited[j] = 1;
            if (seq_next != issued) {
                out.why = "stream_drain's stage count differs from the stages issued";
                return out;
            }
            for (uint32_t j = 0; j < issued; ++j)
                if (!waited[j]) {
                    out.why = "a stage still in flight after the bail-out";
                    return out;
                }
            out.rc = 1;
            out.bail_chunk = c;
            return out;
        }
        // ---- pass 1
        uint32_t accv[32], sh[32];
        int32_t P[32], sumP[32];
        for (int lane = 0; lane < 32; ++lane) {
            accv[lane] = 0;
            sh[lane] = 0;
            P[lane] = 0;
            sumP[lane] = 0;
            int32_t mnu = 0, mxu = 0;
            if (all_full) fast_lane_decode<true, kNeedSum>(wa[lane], wb[lane], valid[lane], term[lane], 0xffffffffu, accv[lane], sh[lane], P[lane], sumP[lane], mnu, mxu);
            else fast_lane_decode<false, kNeedSum>(wa[lane], wb[lane], valid[lane], term[lane], 0xffffffffu, accv[lane], sh[lane], P[lane], sumP[lane], mnu, mxu);
        }
        uint32_t prev_acc[32], prev_sh[32];
        for (int lane = 0; lane < 32; ++lane) {
            prev_acc[lane] = lane == 0 ? carry_acc : accv[lane - 1];
            prev_sh[lane] = lane == 0 ? carry_sh : sh[lane - 1];
        }
        carry_acc = accv[31];
        carry_sh = sh[31];
        for (int lane = 0; lane < 32; ++lane) {
            if (n[lane] > 0 && prev_sh[lane] != 0) {
                const int32_t dlt = head_delta(wa[lane].x, term[lane], prev_acc[lane], prev_sh[lane]);
                P[lane] += dlt;
                sumP[lane] += dlt * static_cast<int32_t>(n[lane]);
            }
            // the lane's totals in 64 bits from its true values: int32 P / sumP must not have wrapped
            std::vector<int32_t> xs;
            lane_values(wa[lane], wb[lane], valid[lane], term[lane], prev_acc[lane], prev_sh[lane], xs);
            int64_t p64 = 0, s64 = 0;
            for (int32_t x : xs) {
                p64 += x;
                s64 += p64;
            }
            if (xs.size() != n[lane] || p64 != P[lane] || s64 != sumP[lane] || s64 > kSumPBound || -s64 > kSumPBound) {
                out.why = "a lane's int32 P / sumP differ from its 64-bit sums";
                return out;
            }
        }
        // ---- warp scan of (n, q, r), inclusive, as the shuffles compute it
        uint32_t n_in[32];
        int64_t q_in[32], r_in[32];
        for (int lane = 0; lane < 32; ++lane) {
            n_in[lane] = n[lane];
            q_in[lane] = P[lane];
            r_in[lane] = sumP[lane];
        }
        for (int s = 1; s < 32; s <<= 1) {
            uint32_t on[32];
            int64_t oq[32], orr[32];
            for (int lane = 0; lane < 32; ++lane) {
                on[lane] = lane >= s ? n_in[lane - s] : n_in[lane];
                oq[lane] = lane >= s ? q_in[lane - s] : q_in[lane];
                orr[lane] = lane >= s ? r_in[lane - s] : r_in[lane];
            }
            for (int lane = s; lane < 32; ++lane) {
                r_in[lane] = wadd(wadd(orr[lane], r_in[lane]), wmul(n_in[lane], oq[lane]));  // current lane is B: nB * qA
                q_in[lane] = wadd(q_in[lane], oq[lane]);
                n_in[lane] += on[lane];
            }
        }
        // ---- pass 2: the true values of every lane's rows
        for (int lane = 0; lane < 32; ++lane) {
            const uint32_t n_ex = n_in[lane] - n[lane];
            const int64_t q_ex = lane == 0 ? 0 : q_in[lane - 1], r_ex = lane == 0 ? 0 : r_in[lane - 1];
            int64_t D = wadd(D0, q_ex);
            int64_t v = wadd(wadd(V0, wmul(n_ex, D0)), r_ex);
            std::vector<int32_t> xs;
            lane_values(wa[lane], wb[lane], valid[lane], term[lane], prev_acc[lane], prev_sh[lane], xs);
            uint32_t row = row_base + n_ex;
            for (int32_t x : xs) {
                D = wadd(D, x);
                v = wadd(v, D);
                if (row < out.vals.size()) out.vals[row] = v;
                ++row;
            }
        }
        // ---- carries to the next chunk; stream_release
        V0 = wadd(wadd(V0, wmul(n_in[31], D0)), r_in[31]);
        D0 = wadd(D0, q_in[31]);
        row_base += n_in[31];
        if ((c % kChunksPerStage) == kChunksPerStage - 1 || c == nchunks - 1) {
            if (k + kStages < nstages) {
                if (k + kStages != issued) {
                    out.why = "stages issued out of order";
                    return out;
                }
                ++issued;
            }
        }
    }
    out.vals.resize(std::min<size_t>(out.vals.size(), pg.count));
    out.rc = (row_base == pg.count && carry_sh == 0) ? 0 : 2;
    return out;
}

// A page: first difference d1, then the second differences `sd`, its body starting at byte body_start of its aligned copy.
static Page make_page(uint32_t body_start, int64_t first, int64_t d1, const std::vector<int64_t> &sd) {
    Page pg;
    pg.body_start = body_start;
    pg.first = first;
    put_varint(pg.body, d1);
    for (int64_t x : sd) put_varint(pg.body, x);
    pg.count = static_cast<uint32_t>(sd.size()) + 2;
    return pg;
}

static long pages = 0;

// decodes the page both ways; want_bail_chunk: the chunk whose wide check must fire (-1: none)
static bool check(const Page &pg, int64_t want_bail_chunk, const char *what) {
    std::vector<int64_t> want;
    if (!plain_decode(pg, want)) {
        std::printf("FAIL %s: the page itself is malformed\n", what);
        return false;
    }
    for (uint8_t garbage : {static_cast<uint8_t>(0xff), static_cast<uint8_t>(0x00), static_cast<uint8_t>(0x80)}) {
        const Outcome o = dod_page_emulated(pg, garbage);
        ++pages;
        const bool ok = want_bail_chunk >= 0 ? (o.rc == 1 && o.bail_chunk == want_bail_chunk) : (o.rc == 0 && o.vals == want);
        if (!ok) {
            size_t bad = 0;
            while (bad < want.size() && bad < o.vals.size() && o.vals[bad] == want[bad]) ++bad;
            std::printf("FAIL %s: body_start=%u len=%zu count=%u garbage=0x%02x rc=%d bail_chunk=%lld (want %lld) %s first wrong row %zu\n", what,
                        pg.body_start, pg.body.size(), pg.count, garbage, o.rc, static_cast<long long>(o.bail_chunk),
                        static_cast<long long>(want_bail_chunk), o.why, bad);
            return false;
        }
        // a row count that does not match the body must not pass
        if (want_bail_chunk < 0) {
            Page wrong = pg;
            wrong.count += 1;
            if (dod_page_emulated(wrong, garbage).rc == 0) {
                std::printf("FAIL %s: accepted a wrong row count\n", what);
                return false;
            }
        }
    }
    return true;
}

static int64_t first_diff_of_width(int w) {  // the smallest positive first difference whose varint takes w bytes
    return w == 1 ? 5 : (w == 10 ? (1ll << 62) + 12345 : (1ll << (7 * (w - 1) - 1)));
}

int main() {
    std::mt19937_64 rng(20261016);
    auto narrow = [&](int L) -> int64_t {  // a random second difference whose varint takes exactly L <= 3 bytes
        const int64_t lo = L == 1 ? 0 : (1ll << (7 * (L - 1) - 1)), hi = (1ll << (7 * L - 1)) - 1;
        const int64_t m = lo + static_cast<int64_t>(rng() % static_cast<uint64_t>(hi - lo + 1));
        return (rng() & 1) ? m : -m - 1 + (L == 1 || m > lo ? 1 : 0);
    };
    for (uint32_t bs = 0; bs < 16; ++bs) {
        for (int w1 = 1; w1 <= 10; ++w1) {
            const int64_t d1 = (rng() & 1) ? first_diff_of_width(w1) : -first_diff_of_width(w1) - 1;  // w1 bytes either way
            const int64_t first = static_cast<int64_t>(rng());
            // a body of the first difference alone (2 rows: the len == 0 exit; the writer itself makes such a list constant-step)
            if (!check(make_page(bs, first, d1, {}), -1, "first difference only")) return 1;
            // 1-byte second differences, stream lengths at and around the lane, chunk and stage edges
            for (uint32_t len : {1u, 2u, 31u, 32u, 33u, 1023u, 1024u, 1025u, 2047u, 2048u, 2049u, 4095u, 4096u, 4097u, 6200u}) {
                std::vector<int64_t> sd(len);
                for (auto &x : sd) x = narrow(1);
                if (!check(make_page(bs, first, d1, sd), -1, "1-byte second differences")) return 1;
            }
            // random 1-3 byte mixes
            for (int t = 0; t < 4; ++t) {
                std::vector<int64_t> sd(1500 + rng() % 1500);
                for (auto &x : sd) x = narrow(1 + static_cast<int>(rng() % 3));
                if (!check(make_page(bs, first, d1, sd), -1, "1-3 byte second differences")) return 1;
            }
            // a 3-byte second difference across every lane edge (and every chunk and stage edge): its first byte at 32k - 2,
            // 32k - 1 or 32k of the aligned copy, 1-byte ones in between
            for (int at = -2; at <= 0; ++at) {
                std::vector<int64_t> sd;
                uint32_t cur = (bs + w1) & 15u;  // aligned position of the next second difference
                for (uint32_t k = 1; k <= 130; ++k) {
                    const uint32_t target = 32 * k + at;
                    for (; cur < target; ++cur) sd.push_back(narrow(1));
                    if (cur != target) continue;
                    sd.push_back(narrow(3));
                    cur += 3;
                }
                for (int t = 0; t < 5; ++t) sd.push_back(narrow(1));
                if (!check(make_page(bs, first, d1, sd), -1, "3-byte second differences across every lane edge")) return 1;
            }
            // a 4-byte second difference: the wide check fires in the chunk of its third byte and not before
            for (uint32_t target : {5u, 31u, 32u, 33u, 1022u, 1023u, 1024u, 2046u, 2047u, 2048u, 3000u, 4094u, 4096u}) {
                std::vector<int64_t> sd;
                uint32_t cur = (bs + w1) & 15u;
                if (target < cur) continue;
                for (; cur < target; ++cur) sd.push_back(narrow(1));
                sd.push_back((rng() & 1) ? (1ll << 20) : -(1ll << 20) - 1);
                for (int t = 0; t < 700; ++t) sd.push_back(narrow(1 + static_cast<int>(rng() % 3)));
                const Page pg = make_page(bs, first, d1, sd);
                if (!check(pg, (target + 2) / kFastChunkBytes, "4-byte second difference")) return 1;
            }
        }
    }
    // int32 P / sumP at the widest lanes the wide check admits: k 3-byte varints of the largest magnitude, then 1-byte ones
    // of the largest magnitude, same sign, repeated (dod_page_emulated compares every lane with its 64-bit sums)
    for (int k = 0; k <= 11; ++k) {
        for (int sign : {1, -1}) {
            for (uint32_t bs = 0; bs < 16; bs += 5) {
                std::vector<int64_t> sd;
                while (sd.size() < 3000) {
                    for (int i = 0; i < k; ++i) sd.push_back(sign > 0 ? (1ll << 20) - 1 : -(1ll << 20));
                    for (int i = 0; i < 32 - 3 * k; ++i) sd.push_back(sign > 0 ? 63 : -64);
                }
                if (!check(make_page(bs, 0, 1, sd), -1, "largest narrow lanes")) return 1;
            }
        }
    }
    std::printf("OK %ld pages\n", pages);
    return 0;
}
