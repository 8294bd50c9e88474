// dense_page.cuh -- the bit-plane form of a narrow delta page (DESIGN.md 3.3).
//
// A field page the express lane sums (EncodeTypeDelta, varints of at most 3 bytes, values v_0 .. v_{n-1}) whose values span
// b <= 32 bits is rewritten at admission as u_i = v_i - m (m = the smallest value) in bit planes: one plane per set bit of b,
// widest first, the plane of width w holding bits [dense_plane_shift(b, w), + w) of every u_i.  Row i sits at bit i * w of the
// plane, in little-endian 32-bit words, so no field crosses a word; each plane is zero-padded to 16 bytes.  The page sum is then
//     sum v = n * m + sum over planes of 2^shift * (sum of the plane's fields)
// and a 16-byte piece of a plane sums its fields with a popcount or a byte dot product per word: no varint decode.
//
// Plain functions of one lane's registers, compiled for the device (scan_kernels.cu) and for the host
// (tests/native/dense_page_test.cc checks them against an exact 128-bit sum).
#pragma once

#include <cstdint>

#include "lane_decode.cuh"

namespace bydb {

// One page's dense form, in a table parallel to the part's DevCol table (same index).  n == 0: the page has none.
struct DevDense {
    const uint8_t *planes;  // 16-byte aligned plane stream of plane_bytes bytes (unused when b == 0)
    int64_t min;            // m (a float64 page: its decimal integers)
    uint32_t n;             // rows of the page; 0 = no dense form
    uint32_t plane_bytes;   // dense_stream_bytes(n, b): a multiple of 16
    int16_t exp;            // decimal exponent of a float64 page
    uint8_t b;              // bit length of max - m, 0 .. 32
    uint8_t pad[5];
};
static_assert(sizeof(DevDense) == 32, "DevDense layout");

constexpr uint32_t kDenseMaxRows = 65536;  // larger blocks keep their varint pages (n * 32 stays far from 2^32 bits)
constexpr int kDensePlanes = 6;            // widths 32, 16, 8, 4, 2, 1

BYDB_LANE_FN uint32_t dense_width(int k) { return 32u >> k; }
// bytes of a plane of width w over n rows: n * w bits in whole 32-bit words, padded to 16 bytes
BYDB_LANE_FN uint32_t dense_plane_bytes(uint32_t n, uint32_t w) { return (n * w + 127u) / 128u * 16u; }
// lowest bit of u the plane of width w holds: the set bits of b above w come first
BYDB_LANE_FN uint32_t dense_plane_shift(uint32_t b, uint32_t w) { return b & ~(2u * w - 1u); }
// end offsets of the planes in the stream, widest first (an absent width ends where the one before it does);
// end[kDensePlanes - 1] is the stream's length
BYDB_LANE_FN void dense_plane_ends(uint32_t n, uint32_t b, uint32_t end[kDensePlanes]) {
    uint32_t e = 0;
#pragma unroll
    for (int k = 0; k < kDensePlanes; ++k) {
        if (b & dense_width(k)) e += dense_plane_bytes(n, dense_width(k));
        end[k] = e;
    }
}
BYDB_LANE_FN uint32_t dense_stream_bytes(uint32_t n, uint32_t b) {
    uint32_t end[kDensePlanes];
    dense_plane_ends(n, b, end);
    return end[kDensePlanes - 1];
}

// the sum of the w-bit fields of one 32-bit word
template <int W>
BYDB_LANE_FN uint32_t dense_word_sum(uint32_t x) {
    if (W == 16) return (x & 0xffffu) + (x >> 16);
    if (W == 8) return static_cast<uint32_t>(dp4a_us(x, 0x01010101u, 0));
    if (W == 4) return static_cast<uint32_t>(dp4a_us(x & 0x0f0f0f0fu, 0x01010101u, dp4a_us((x >> 4) & 0x0f0f0f0fu, 0x01010101u, 0)));
    if (W == 2) return lane_popc(x) + lane_popc(x & 0xaaaaaaaau);
    return lane_popc(x);  // W == 1
}
template <int W>
BYDB_LANE_FN uint64_t dense_piece_fields(const uint4 &v) {
    if (W == 32) return static_cast<uint64_t>(v.x) + v.y + v.z + v.w;
    return dense_word_sum<W>(v.x) + dense_word_sum<W>(v.y) + dense_word_sum<W>(v.z) + dense_word_sum<W>(v.w);
}
// The contribution of the 16-byte piece at stream offset `off` to sum u: its fields times 2^shift of its plane.  A piece at or
// beyond the stream's end (bytes a stage holds from an earlier copy) adds nothing.
BYDB_LANE_FN uint64_t dense_piece_sum(const uint4 &v, uint32_t off, const uint32_t end[kDensePlanes], uint32_t b) {
    if (off < end[0]) return dense_piece_fields<32>(v) << dense_plane_shift(b, 32);
    if (off < end[1]) return dense_piece_fields<16>(v) << dense_plane_shift(b, 16);
    if (off < end[2]) return dense_piece_fields<8>(v) << dense_plane_shift(b, 8);
    if (off < end[3]) return dense_piece_fields<4>(v) << dense_plane_shift(b, 4);
    if (off < end[4]) return dense_piece_fields<2>(v) << dense_plane_shift(b, 2);
    if (off < end[5]) return dense_piece_fields<1>(v) << dense_plane_shift(b, 1);
    return 0;
}

// word q of the plane of width w (b: the page's bit length) over the rows' u values
BYDB_LANE_FN uint32_t dense_encode_word(const uint32_t *u, uint32_t n, uint32_t b, uint32_t w, uint32_t q) {
    const uint32_t per = 32u / w, s = dense_plane_shift(b, w), mask = low_bits(w);
    uint32_t x = 0;
    for (uint32_t i = 0; i < per; ++i) {
        const uint32_t r = q * per + i;
        if (r < n) x |= ((u[r] >> s) & mask) << (i * w);
    }
    return x;
}

}  // namespace bydb
