// index_kernels.cu -- the block index of a measure part decoded ON THE DEVICE (SURVEY.md 8f row 1).
//
// Replaces, at part admission, the host-side libzstd + parse of part_dir.cc:
//   meta.bin     = zstd(concat primaryBlockMetadata), 40 B records                   primary_metadata.go:47-83,106-137
//   primary.bin  = one zstd frame per primary block = concat blockMetadata records    part_iter.go:184-208, block_writer.go:247-276
//   blockMetadata / timestampsMetadata / columnFamilyMetadata                         block_metadata.go:133-168,279-293; column_metadata.go:108-122
//   <family>.tfm = per block and family the tag columns' columnFamilyMetadata
// into the flat DevBlock[] / DevCol[] directory the scan kernels read.
//
//   index_meta_kernel      one thread: inflate meta.bin, validate the 40 B records, read every primary frame's declared size
//   index_inflate_kernel   one warp per primary frame: lane 0 runs the RFC 8878 decoder of zstd_dec.cuh
//   index_walk_kernel<0>   one thread per primary block: walk the records -- count blocks / columns, intern the column names
//   index_walk_kernel<1>   the same walk, now writing DevBlock / DevCol at the prefix-summed positions
//   index_order_kernel     one thread per block: global (sid, min timestamp) order (block_metadata.go:323-336), row totals
// Names: columns are interned into a small device table ("f:<field>" / "t:<family>/<tag>"); the host maps the table to the
// context's name ids between the two walks (a few dozen strings -- no page bytes and no index bytes are parsed on the host).
#include "index_kernels.cuh"
#include "scan_kernels.cuh"

#include "../../include/bydb_gpu.h"
#include "zstd_dec.cuh"

namespace bydb {

namespace {

constexpr size_t kIndexWsBytes = (sizeof(zstd::Workspace) + 255u) & ~static_cast<size_t>(255u);
constexpr size_t kIndexScratchStride = kIndexWsBytes + 131072 + 256;  // workspace + one block's worth of literals

struct Cur {
    const uint8_t *p, *end;
    bool bad;
    __device__ size_t left() const { return static_cast<size_t>(end - p); }
    __device__ uint64_t u64be() {
        if (left() < 8) {
            bad = true;
            return 0;
        }
        uint64_t u = 0;
        for (int k = 0; k < 8; ++k) u = (u << 8) | p[k];
        p += 8;
        return u;
    }
    __device__ uint8_t u8() {
        if (left() < 1) {
            bad = true;
            return 0;
        }
        return *p++;
    }
    __device__ uint64_t varu() {  // pkg/encoding/int.go:189-211
        uint64_t x = 0;
        for (unsigned s = 0, i = 0; i < 10; ++i, s += 7) {
            if (p >= end) break;
            const uint8_t b = *p++;
            x |= static_cast<uint64_t>(b & 0x7f) << s;
            if (b < 0x80) return x;
        }
        bad = true;
        return 0;
    }
};

__device__ __forceinline__ bool in_file(uint64_t off, uint64_t size, uint64_t len) { return off <= len && size <= len - off; }

__device__ void set_index_err(const IndexParams &p, uint32_t code, uint32_t where) {
    if (atomicCAS(&p.ctl->err, 0u, code) == 0u) p.ctl->err_where = where;
}

__device__ bool bytes_equal(const uint8_t *a, const uint8_t *b, uint32_t n) {
    for (uint32_t i = 0; i < n; ++i)
        if (a[i] != b[i]) return false;
    return true;
}

// -> local name id (index into the device name table); kind 'f' = field, 't' = tag of family `fam`
__device__ uint32_t intern_name(const IndexParams &p, uint8_t kind, uint32_t fam, const uint8_t *name, uint32_t len) {
    if (len > kIndexNameMax) return 0xffffffffu;
    for (;;) {
        const uint32_t n = *reinterpret_cast<volatile uint32_t *>(&p.ctl->n_names);
        for (uint32_t i = 0; i < n; ++i) {
            const IndexName &e = p.names[i];
            if (e.kind == kind && e.fam == fam && e.len == len && bytes_equal(e.bytes, name, len)) return i;
        }
        // append under the table lock (callers are single lanes of distinct warps: spinning cannot deadlock a warp)
        if (atomicCAS(&p.ctl->name_lock, 0u, 1u) != 0u) continue;
        const uint32_t n2 = *reinterpret_cast<volatile uint32_t *>(&p.ctl->n_names);
        uint32_t id = 0xffffffffu;
        if (n2 == n) {
            if (n < kIndexMaxNames) {
                IndexName &e = p.names[n];
                e.kind = kind;
                e.fam = static_cast<uint8_t>(fam);
                e.len = static_cast<uint8_t>(len);
                for (uint32_t i = 0; i < len; ++i) e.bytes[i] = name[i];
                __threadfence();
                *reinterpret_cast<volatile uint32_t *>(&p.ctl->n_names) = n + 1;
                id = n;
            } else {
                id = 0xfffffffeu;  // table full
            }
        }
        __threadfence();
        atomicExch(&p.ctl->name_lock, 0u);
        if (id != 0xffffffffu) return id;
        // somebody appended meanwhile: look again
    }
}

// Consecutive blocks usually share a schema: position -> (family, bytes, id), like part_dir.cc's positional cache.  A part
// holds the series of several measures, so a neighbouring block may carry the same tag name at the same position in
// another family: a hit needs the family too.
struct NameCache {
    const uint8_t *ptr[kIndexCacheSlots];
    uint32_t len[kIndexCacheSlots];
    uint32_t id[kIndexCacheSlots];
    uint8_t fam[kIndexCacheSlots];  // tags: slot in IndexParams::families (< 251); fields: 0
};
__device__ uint32_t resolve_name(const IndexParams &p, NameCache &nc, uint32_t pos, uint8_t kind, uint32_t fam, const uint8_t *name, uint32_t len) {
    if (pos < kIndexCacheSlots && nc.ptr[pos] && nc.fam[pos] == fam && nc.len[pos] == len && bytes_equal(nc.ptr[pos], name, len)) return nc.id[pos];
    const uint32_t id = intern_name(p, kind, fam, name, len);
    if (pos < kIndexCacheSlots) {
        nc.ptr[pos] = name;
        nc.len[pos] = len;
        nc.id[pos] = id;
        nc.fam[pos] = static_cast<uint8_t>(fam);
    }
    return id;
}

}  // namespace

// ------------------------------------------------------------------------------------------------ meta.bin
// phase 0: the declared size of the meta frame; phase 1: inflate + validate + the primary frames' declared sizes
__global__ void index_meta_kernel(const __grid_constant__ IndexParams p, int phase) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    if (phase == 0) {
        const int64_t n = zstd::frame_content_size(p.meta, static_cast<int64_t>(p.meta_len));
        if (n < 0 || (n % 40) != 0) {
            set_index_err(p, kIdxBadMeta, 0);
            return;
        }
        p.ctl->meta_raw = static_cast<uint64_t>(n);
        return;
    }
    zstd::Workspace *ws = reinterpret_cast<zstd::Workspace *>(p.scratch);
    uint8_t *lit = p.scratch + kIndexWsBytes;
    const int64_t got = zstd::decode_frame(ws, p.meta, static_cast<int64_t>(p.meta_len), p.meta_raw, static_cast<int64_t>(p.meta_raw_cap), lit);
    if (got < 0 || static_cast<uint64_t>(got) != p.meta_raw_cap) {
        set_index_err(p, kIdxBadMeta, 1);
        return;
    }
    const uint32_t np = static_cast<uint32_t>(p.meta_raw_cap / 40);
    uint64_t total = 0, prev_sid = 0;
    for (uint32_t i = 0; i < np; ++i) {
        Cur c{p.meta_raw + 40ull * i, p.meta_raw + 40ull * (i + 1), false};
        const uint64_t sid = c.u64be();
        (void)c.u64be();
        (void)c.u64be();
        const uint64_t off = c.u64be(), size = c.u64be();
        if (!in_file(off, size, p.primary_len) || (i > 0 && sid < prev_sid)) {  // primary_metadata.go:127-134
            set_index_err(p, kIdxBadMeta, 2 + i);
            return;
        }
        prev_sid = sid;
        const int64_t raw = zstd::frame_content_size(p.primary + off, static_cast<int64_t>(size));
        if (raw < 0 || raw > (64ll << 20)) {
            set_index_err(p, kIdxBadFrame, i);
            return;
        }
        p.pb[i].off = off;
        p.pb[i].size = size;
        p.pb[i].raw_off = total;
        p.pb[i].raw_len = static_cast<uint64_t>(raw);
        total += (static_cast<uint64_t>(raw) + 15u) & ~15ull;
    }
    p.ctl->n_primary = np;
    p.ctl->raw_total = total;
}

// ------------------------------------------------------------------------------------------------ primary.bin frames
__global__ void index_inflate_kernel(const __grid_constant__ IndexParams p) {
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if ((threadIdx.x & 31) != 0 || w >= p.n_primary) return;
    uint8_t *scratch = p.scratch + static_cast<size_t>(w) * kIndexScratchStride;
    zstd::Workspace *ws = reinterpret_cast<zstd::Workspace *>(scratch);
    const IndexPrimary pb = p.pb[w];
    const int64_t got = zstd::decode_frame(ws, p.primary + pb.off, static_cast<int64_t>(pb.size), p.raw + pb.raw_off, static_cast<int64_t>(pb.raw_len),
                                           scratch + kIndexWsBytes);
    if (got < 0 || static_cast<uint64_t>(got) != pb.raw_len) set_index_err(p, kIdxBadFrame, w);
}

// ------------------------------------------------------------------------------------------------ record walk
template <bool kFill>
__global__ void index_walk_kernel(const __grid_constant__ IndexParams p) {
    const uint32_t w = blockIdx.x;  // one walker per CTA (lane 0): the name table's spin lock never has two holders in a warp
    if (threadIdx.x != 0 || w >= p.n_primary) return;
    const IndexPrimary pb = p.pb[w];
    Cur c{p.raw + pb.raw_off, p.raw + pb.raw_off + pb.raw_len, false};
    NameCache fcache, tcache;
    for (uint32_t i = 0; i < kIndexCacheSlots; ++i) fcache.ptr[i] = tcache.ptr[i] = nullptr;
    uint32_t nb = 0, nc = 0;
    uint64_t bi = kFill ? p.pb[w].block_base : 0, ci = kFill ? p.pb[w].col_base : 0;
    uint64_t prev_sid = 0;
    int64_t prev_min = 0;
    while (c.p < c.end) {
        DevBlock b;
        b.sid = c.u64be();
        (void)c.varu();  // uncompressedSizeBytes: accounting only
        const uint64_t count = c.varu();
        b.ts_off = c.varu();
        const uint64_t ts_size = c.varu();
        b.ts_min = static_cast<int64_t>(c.u64be());
        b.ts_max = static_cast<int64_t>(c.u64be());
        const uint8_t enc = c.u8();
        const uint64_t ver_off = c.varu();
        b.ver_first = static_cast<int64_t>(c.u64be());
        b.ver_enc = c.u8();
        if (c.bad || count == 0 || count > 0x7fffffffu || ts_size > 0xffffffffu || ver_off > ts_size || !in_file(b.ts_off, ts_size, p.ts_len)) {
            set_index_err(p, kIdxBadBlock, w);
            return;
        }
        if (enc < 5 || enc > 8 || b.ver_enc < 1 || b.ver_enc > 4) {  // encoding.go:87-130
            set_index_err(p, kIdxBadEnc, w);
            return;
        }
        if (nb > 0 && (b.sid < prev_sid || (b.sid == prev_sid && b.ts_min < prev_min))) {
            set_index_err(p, kIdxOrder, w);
            return;
        }
        prev_sid = b.sid;
        prev_min = b.ts_min;
        b.ts_enc = static_cast<uint8_t>(enc - 4);
        b.count = static_cast<uint32_t>(count);
        b.ts_size = static_cast<uint32_t>(ts_size);
        b.ver_off = static_cast<uint32_t>(ver_off);
        b.col_begin = static_cast<uint32_t>(ci);
        b.pad = 0;
        // tag families of the block: (name, off, size) into <name>.tfm
        const uint64_t nfam = c.varu();
        if (c.bad || nfam > 16) {
            set_index_err(p, nfam > 16 ? kIdxTooManyFamilies : kIdxBadBlock, w);
            return;
        }
        uint32_t fam_slot[16];
        uint64_t fam_off[16], fam_size[16];
        for (uint64_t f = 0; f < nfam; ++f) {
            const uint64_t nl = c.varu();
            if (c.bad || c.left() < nl) {
                set_index_err(p, kIdxBadBlock, w);
                return;
            }
            const uint8_t *np = c.p;
            c.p += nl;
            uint32_t slot = 0xffffffffu;
            for (uint32_t k = 0; k < p.n_families; ++k)
                if (p.families[k].name_len == nl && bytes_equal(p.families[k].name, np, static_cast<uint32_t>(nl))) slot = k;
            fam_slot[f] = slot;
            fam_off[f] = c.varu();
            fam_size[f] = c.varu();
        }
        // fields: columnFamilyMetadata.unmarshal, column_metadata.go:108-122
        const uint64_t nf = c.varu();
        uint32_t ncols_blk = 0;
        for (uint64_t i = 0; i < nf && !c.bad; ++i) {
            const uint64_t nl = c.varu();
            if (c.bad || c.left() < nl) {
                c.bad = true;
                break;
            }
            const uint8_t *np = c.p;
            c.p += nl;
            DevCol col;
            col.value_type = c.u8();
            col.off = c.varu();
            const uint64_t size = c.varu();
            if (c.bad || size > 0xffffffffu || !in_file(col.off, size, p.fv_len)) {
                set_index_err(p, kIdxBadColumn, w);
                return;
            }
            const uint32_t lid = resolve_name(p, fcache, static_cast<uint32_t>(i), 'f', 0, np, static_cast<uint32_t>(nl));
            if (lid >= kIndexMaxNames) {
                set_index_err(p, kIdxNames, w);
                return;
            }
            if (kFill) {
                col.size = static_cast<uint32_t>(size);
                col.name_id = p.name_map[lid];
                col.file_id = 1;
                p.cols[ci] = col;
            }
            ++ci;
            ++ncols_blk;
        }
        if (c.bad) {
            set_index_err(p, kIdxBadBlock, w);
            return;
        }
        uint32_t tag_pos = 0;
        for (uint64_t f = 0; f < nfam; ++f) {
            if (fam_slot[f] == 0xffffffffu || !in_file(fam_off[f], fam_size[f], p.families[fam_slot[f]].tfm_len)) {
                set_index_err(p, kIdxFamily, w);
                return;
            }
            const IndexFamily &fam = p.families[fam_slot[f]];
            Cur t{fam.tfm + fam_off[f], fam.tfm + fam_off[f] + fam_size[f], false};
            const uint64_t ncf = t.varu();
            for (uint64_t i = 0; i < ncf && !t.bad; ++i, ++tag_pos) {
                const uint64_t nl = t.varu();
                if (t.bad || t.left() < nl) {
                    t.bad = true;
                    break;
                }
                const uint8_t *np = t.p;
                t.p += nl;
                DevCol col;
                col.value_type = t.u8();
                col.off = t.varu();
                const uint64_t size = t.varu();
                if (t.bad || size > 0xffffffffu || !in_file(col.off, size, fam.tf_len)) {
                    set_index_err(p, kIdxBadColumn, w);
                    return;
                }
                const uint32_t lid = resolve_name(p, tcache, tag_pos, 't', fam_slot[f], np, static_cast<uint32_t>(nl));
                if (lid >= kIndexMaxNames) {
                    set_index_err(p, kIdxNames, w);
                    return;
                }
                if (kFill) {
                    col.size = static_cast<uint32_t>(size);
                    col.name_id = p.name_map[lid];
                    col.file_id = fam.file_id;
                    p.cols[ci] = col;
                }
                ++ci;
                ++ncols_blk;
            }
            if (t.bad) {
                set_index_err(p, kIdxBadColumn, w);
                return;
            }
        }
        if (ncols_blk > 0xffff) {
            set_index_err(p, kIdxBadBlock, w);
            return;
        }
        if (kFill) {
            b.n_cols = static_cast<uint16_t>(ncols_blk);
            p.blocks[bi] = b;
        }
        ++bi;
        ++nb;
        nc += ncols_blk;
    }
    if (!kFill) {
        p.pb[w].n_blocks = nb;
        p.pb[w].n_cols = nc;
    }
}

// global order across primary blocks + the part's totals
__global__ void index_order_kernel(const __grid_constant__ IndexParams p) {
    const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= p.n_blocks) return;
    const DevBlock &b = p.blocks[i];
    if (i > 0) {
        const DevBlock &pre = p.blocks[i - 1];
        if (b.sid < pre.sid || (b.sid == pre.sid && b.ts_min < pre.ts_min)) set_index_err(p, kIdxOrder, static_cast<uint32_t>(i));
    }
    atomicAdd(&p.ctl->total_rows, static_cast<unsigned long long>(b.count));
    atomicMax(&p.ctl->max_block_rows, b.count);
    atomicMin(&p.ctl->min_ts, b.ts_min);
    atomicMax(&p.ctl->max_ts, b.ts_max);
}

size_t index_ws_bytes() { return kIndexWsBytes; }
size_t index_scratch_stride() { return kIndexScratchStride; }

void launch_index_meta(const IndexParams &p, int phase, cudaStream_t s) { index_meta_kernel<<<1, 32, 0, s>>>(p, phase); }
void launch_index_inflate(const IndexParams &p, cudaStream_t s) {
    if (p.n_primary == 0) return;
    const unsigned warps_per_cta = 4;
    index_inflate_kernel<<<(p.n_primary + warps_per_cta - 1) / warps_per_cta, warps_per_cta * 32, 0, s>>>(p);
}
void launch_index_walk(const IndexParams &p, bool fill, cudaStream_t s) {
    if (p.n_primary == 0) return;
    // the walk is sequential per primary block (variable-length records): one single-lane CTA each, spread over the SMs
    if (fill) index_walk_kernel<true><<<p.n_primary, 32, 0, s>>>(p);
    else index_walk_kernel<false><<<p.n_primary, 32, 0, s>>>(p);
}
void launch_index_order(const IndexParams &p, cudaStream_t s) {
    if (p.n_blocks == 0) return;
    index_order_kernel<<<static_cast<unsigned>((p.n_blocks + 255) / 256), 256, 0, s>>>(p);
}

void preload_index_kernels() {
    cudaFuncAttributes a;
    cudaFuncGetAttributes(&a, index_meta_kernel);
    cudaFuncGetAttributes(&a, index_inflate_kernel);
    cudaFuncGetAttributes(&a, index_walk_kernel<true>);
    cudaFuncGetAttributes(&a, index_walk_kernel<false>);
    cudaFuncGetAttributes(&a, index_order_kernel);
    cudaGetLastError();
}

}  // namespace bydb
