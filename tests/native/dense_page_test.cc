// Host build of the dense page form (skywalking-banyandb_b200/csrc/dense_page.cuh): pages are encoded with dense_encode_word and
// summed with dense_piece_sum exactly as the express lane walks them -- 4 KB units, lane l taking the 16-byte pieces l, l + 32,
// ... of a unit, the bytes of the last unit beyond the stream left stale (0xff) -- and n * m + sum is compared with the exact
// 128-bit sum of the values.  Every bit length b from 0 to 32, row counts from 1 to 8448, m at both ends of int64.
// Built and run by tests/test_dense_page_native.py with g++ (the CUDA toolkit headers only provide uint4).
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

#include "dense_page.cuh"

using namespace bydb;

constexpr uint32_t kUnit = 4096;  // the express lane's stage (kExpressStageBytes)
static int failures = 0;

static void check_page(const std::vector<uint32_t> &u, uint32_t b, int64_t m) {
    const uint32_t n = static_cast<uint32_t>(u.size());
    uint32_t end[kDensePlanes];
    dense_plane_ends(n, b, end);
    const uint32_t bytes = end[kDensePlanes - 1];
    if (bytes != dense_stream_bytes(n, b) || bytes % 16) {
        std::printf("FAIL stream size n=%u b=%u\n", n, b);
        ++failures;
        return;
    }
    // the plane stream, as the write pass lays it out
    const uint32_t units = (bytes + kUnit - 1) / kUnit;
    std::vector<uint8_t> stream(static_cast<size_t>(units) * kUnit, 0xff);
    uint32_t at = 0;
    for (int k = 0; k < kDensePlanes; ++k) {
        const uint32_t w = dense_width(k);
        if (!(b & w)) continue;
        const uint32_t words = dense_plane_bytes(n, w) / 4;
        for (uint32_t q = 0; q < words; ++q) {
            const uint32_t x = dense_encode_word(u.data(), n, b, w, q);
            std::memcpy(&stream[at + 4 * q], &x, 4);
        }
        at += words * 4;
    }
    if (at != bytes) {
        std::printf("FAIL layout n=%u b=%u\n", n, b);
        ++failures;
        return;
    }
    // the express lane's walk: per unit, per lane, per piece
    uint64_t lanes[32] = {};
    for (uint32_t j = 0; j < units; ++j)
        for (uint32_t lane = 0; lane < 32; ++lane)
            for (uint32_t q = 0; q < kUnit / 512; ++q) {
                const uint32_t pc = lane + 32 * q;
                uint4 v;
                std::memcpy(&v, &stream[static_cast<size_t>(j) * kUnit + 16 * pc], 16);
                lanes[lane] += dense_piece_sum(v, j * kUnit + 16 * pc, end, b);
            }
    uint64_t U = 0;
    for (uint64_t x : lanes) U += x;
    __int128 got = static_cast<__int128>(m) * n + static_cast<__int128>(U);
    __int128 want = 0;
    for (uint32_t x : u) want += static_cast<__int128>(m) + x;
    if (got != want) {
        std::printf("FAIL sum n=%u b=%u m=%lld\n", n, b, static_cast<long long>(m));
        ++failures;
    }
}

int main() {
    std::mt19937_64 rng(20261017);
    std::vector<uint32_t> counts;
    for (uint32_t n = 1; n <= 70; ++n) counts.push_back(n);
    for (uint32_t n : {127u, 128u, 129u, 255u, 256u, 257u, 1023u, 1024u, 1025u, 2047u, 2048u, 2049u, 4095u, 4096u, 4097u, 8191u, 8192u, 8193u, 8447u, 8448u})
        counts.push_back(n);
    for (int i = 0; i < 40; ++i) counts.push_back(1 + static_cast<uint32_t>(rng() % 8448));
    const int64_t mins[] = {0, -123456789, 1700000000000LL, INT64_MIN, INT64_MIN + 1, INT64_MAX};
    long pages = 0;
    for (uint32_t b = 0; b <= 32; ++b) {
        const uint64_t top = b ? ((1ull << b) - 1) : 0;  // largest u of the page: its bit length is exactly b
        for (uint32_t n : counts) {
            for (int64_t m0 : mins) {
                // m + top must stay in int64
                const int64_t m = m0 > INT64_MAX - static_cast<int64_t>(top) ? INT64_MAX - static_cast<int64_t>(top) : m0;
                std::vector<uint32_t> u(n);
                const int kind = static_cast<int>(rng() % 3);
                for (uint32_t i = 0; i < n; ++i) {
                    const uint64_t r = rng();
                    u[i] = static_cast<uint32_t>(kind == 0 ? (top ? r % (top + 1) : 0) : kind == 1 ? top - (top ? r % (top / 8 + 1) : 0) : (top ? r & top : 0));
                }
                u[rng() % n] = static_cast<uint32_t>(top);
                u[rng() % n] = 0;
                if (n == 1) u[0] = 0;  // a 1-row page spans nothing
                check_page(u, n == 1 ? 0 : b, m);
                ++pages;
            }
        }
    }
    if (failures) {
        std::printf("FAILED %d of %ld pages\n", failures, pages);
        return 1;
    }
    std::printf("OK %ld pages\n", pages);
    return 0;
}
