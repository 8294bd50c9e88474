// part_dir.cc -- see part_dir.hpp.
#include "part_dir.hpp"

#include <dlfcn.h>

#include <algorithm>
#include <cstring>
#include <exception>
#include <mutex>
#include <thread>

#include "../../include/bydb_gpu.h"

namespace bydb {

uint16_t NameTable::intern(const std::string &s) {
    std::lock_guard<std::mutex> lk(mu_);
    auto it = ids_.find(s);
    if (it != ids_.end()) return it->second;
    uint16_t id = static_cast<uint16_t>(ids_.size() + 1);
    ids_.emplace(s, id);
    return id;
}
uint16_t NameTable::find(const std::string &s) const {
    std::lock_guard<std::mutex> lk(mu_);
    auto it = ids_.find(s);
    return it == ids_.end() ? 0 : it->second;
}

// ------------------------------------------------------------------ zstd (pkg/compress/zstd/zstd.go:49-52)
namespace {
using decompress_fn = size_t (*)(void *, size_t, const void *, size_t);
using iserr_fn = unsigned (*)(size_t);
using fcs_fn = unsigned long long (*)(const void *, size_t);
struct Zstd {
    decompress_fn decompress = nullptr;
    iserr_fn is_error = nullptr;
    fcs_fn content_size = nullptr;
    bool ok = false;
};
Zstd &zstd_lib() {
    static Zstd z;
    static std::once_flag once;
    std::call_once(once, [] {
        void *h = dlopen("libzstd.so.1", RTLD_NOW | RTLD_GLOBAL);
        if (!h) return;
        z.decompress = reinterpret_cast<decompress_fn>(dlsym(h, "ZSTD_decompress"));
        z.is_error = reinterpret_cast<iserr_fn>(dlsym(h, "ZSTD_isError"));
        z.content_size = reinterpret_cast<fcs_fn>(dlsym(h, "ZSTD_getFrameContentSize"));
        z.ok = z.decompress && z.is_error && z.content_size;
    });
    return z;
}
}  // namespace

int zstd_decompress(const uint8_t *src, size_t n, std::vector<uint8_t> &dst, std::string &err) {
    Zstd &z = zstd_lib();
    if (!z.ok) {
        err = "libzstd.so.1 not available";
        return BYDB_EIO;
    }
    unsigned long long fcs = z.content_size(src, n);
    if (fcs == static_cast<unsigned long long>(-2)) {
        err = "not a zstd frame";
        return BYDB_EINVAL;
    }
    // a frame of the block index is a primary block (flushed above 128 KiB raw, block_writer.go:247-250) or meta.bin
    // (40 B per primary block): a declared size beyond this bound is a corrupt header, not something to allocate
    const unsigned long long kMaxFrame = std::max<unsigned long long>(64ull << 20, static_cast<unsigned long long>(n) * 1024ull);
    if (fcs != static_cast<unsigned long long>(-1) && fcs > kMaxFrame) {
        err = "zstd frame declares an implausible content size";
        return BYDB_EINVAL;
    }
    size_t cap = fcs == static_cast<unsigned long long>(-1) ? n * 32 + 4096 : static_cast<size_t>(fcs);
    for (int attempt = 0; attempt < 8; ++attempt) {
        dst.resize(cap ? cap : 1);
        size_t r = z.decompress(dst.data(), cap, src, n);
        if (!z.is_error(r)) {
            dst.resize(r);
            return 0;
        }
        if (fcs != static_cast<unsigned long long>(-1)) break;
        cap *= 8;
        if (cap > kMaxFrame) break;
    }
    err = "zstd decompress failed";
    return BYDB_EINVAL;
}

// ------------------------------------------------------------------ byte cursor
namespace {
// [off, off+size) inside a file of `len` bytes, without wrapping in uint64 (a crafted offset must not pass)
inline bool in_file(uint64_t off, uint64_t size, uint64_t len) { return off <= len && size <= len - off; }

struct Cur {
    const uint8_t *p, *end;
    bool bad = false;
    size_t left() const { return static_cast<size_t>(end - p); }
    uint64_t u64be() {
        if (left() < 8) {
            bad = true;
            return 0;
        }
        uint64_t u = 0;
        for (int k = 0; k < 8; ++k) u = (u << 8) | p[k];
        p += 8;
        return u;
    }
    uint8_t u8() {
        if (left() < 1) {
            bad = true;
            return 0;
        }
        return *p++;
    }
    // LEB128 unsigned (pkg/encoding/int.go:189-211); a truncated value marks the cursor bad
    uint64_t varu() {
        uint64_t x = 0;
        for (unsigned s = 0, i = 0; i < 10; ++i, s += 7) {
            if (p >= end) break;
            uint8_t b = *p++;
            x |= static_cast<uint64_t>(b & 0x7f) << s;
            if (b < 0x80) return x;
        }
        bad = true;
        return 0;
    }
    std::string str() {  // pkg/encoding/bytes.go:35-43 DecodeBytes
        uint64_t n = varu();
        if (bad || left() < n) {
            bad = true;
            return {};
        }
        std::string s(reinterpret_cast<const char *>(p), static_cast<size_t>(n));
        p += n;
        return s;
    }
};

const FileImage *find_file(const std::vector<FileImage> &files, const std::string &name) {
    for (const auto &f : files)
        if (f.name == name) return &f;
    return nullptr;
}
}  // namespace

// Parses one decompressed primary block (a run of blockMetadata records) into blocks/cols.
// Column names are resolved through a positional cache first (consecutive blocks usually share a schema),
// so the shared NameTable is only touched on a miss.  A part holds the series of several measures, so
// neighbouring blocks may carry other families: a tag slot hits only for the same family, position and bytes.
namespace {
struct NameSlot {
    std::string raw;
    size_t fam = SIZE_MAX;  // tags: slot in ParseCtx::fam_cache
    uint16_t id = 0;
};
struct ParseCtx {
    const std::vector<FileImage> *files;
    const FileImage *tsf, *fvf;
    NameTable *names;
    std::mutex *names_mu;
    std::vector<std::string> *file_table;  // shared, guarded by names_mu
    std::vector<NameSlot> field_cache;
    std::vector<NameSlot> tag_cache;
    struct FamSlot {
        std::string name;
        const FileImage *tfm = nullptr, *tf = nullptr;
        int file_id = -1;
    };
    std::vector<FamSlot> fam_cache;
};

uint16_t resolve_name(ParseCtx &cx, std::vector<NameSlot> &cache, size_t pos, const char *prefix, size_t fam_slot, const std::string &fam, const uint8_t *p,
                      size_t n) {
    if (pos < cache.size() && cache[pos].fam == fam_slot && cache[pos].raw.size() == n && memcmp(cache[pos].raw.data(), p, n) == 0) return cache[pos].id;
    std::string key(prefix);
    if (!fam.empty()) key += fam + "/";
    key.append(reinterpret_cast<const char *>(p), n);
    uint16_t id;
    {
        std::lock_guard<std::mutex> lk(*cx.names_mu);
        id = cx.names->intern(key);
    }
    if (pos >= cache.size()) cache.resize(pos + 1);
    cache[pos].raw.assign(reinterpret_cast<const char *>(p), n);
    cache[pos].fam = fam_slot;
    cache[pos].id = id;
    return id;
}

int parse_primary_block(ParseCtx &cx, const uint8_t *data, size_t len, std::vector<DevBlock> &blocks, std::vector<DevCol> &cols, std::string &err) {
    Cur c{data, data + len};
    while (c.p < c.end) {
        // blockMetadata.unmarshal, block_metadata.go:133-168 (+ timestampsMetadata :279-293)
        DevBlock b{};
        b.sid = c.u64be();
        (void)c.varu();  // uncompressedSizeBytes: accounting only
        uint64_t count = c.varu();
        b.ts_off = c.varu();
        uint64_t ts_size = c.varu();
        b.ts_min = static_cast<int64_t>(c.u64be());
        b.ts_max = static_cast<int64_t>(c.u64be());
        uint8_t enc = c.u8();
        uint64_t ver_off = c.varu();
        b.ver_first = static_cast<int64_t>(c.u64be());
        b.ver_enc = c.u8();
        if (c.bad || count == 0 || count > 0x7fffffffu || ts_size > 0xffffffffu || ver_off > ts_size || !in_file(b.ts_off, ts_size, cx.tsf->len)) {
            err = "corrupt blockMetadata (timestamps)";
            return BYDB_EINVAL;
        }
        if (enc < 5 || enc > 8 || b.ver_enc < 1 || b.ver_enc > 4) {  // encoding.go:87-130
            err = "unexpected timestamps encode type";
            return BYDB_EINVAL;
        }
        b.ts_enc = static_cast<uint8_t>(enc - 4);
        b.count = static_cast<uint32_t>(count);
        b.ts_size = static_cast<uint32_t>(ts_size);
        b.ver_off = static_cast<uint32_t>(ver_off);
        b.col_begin = static_cast<uint32_t>(cols.size());
        // tag families: name -> dataBlock into <name>.tfm (columnFamilyMetadata of this block)
        uint64_t nfam = c.varu();
        struct Fam {
            size_t slot;
            uint64_t off, size;
        };
        Fam fams[16];
        if (nfam > 16) {
            err = "more than 16 tag families in a block";
            return BYDB_ENOTSUP;
        }
        for (uint64_t i = 0; i < nfam && !c.bad; ++i) {
            uint64_t nl = c.varu();
            if (c.bad || c.left() < nl) {
                c.bad = true;
                break;
            }
            const uint8_t *np = c.p;
            c.p += nl;
            size_t slot = cx.fam_cache.size();
            for (size_t k = 0; k < cx.fam_cache.size(); ++k)
                if (cx.fam_cache[k].name.size() == nl && memcmp(cx.fam_cache[k].name.data(), np, nl) == 0) slot = k;
            if (slot == cx.fam_cache.size()) {
                ParseCtx::FamSlot fs;
                fs.name.assign(reinterpret_cast<const char *>(np), nl);
                fs.tfm = find_file(*cx.files, fs.name + ".tfm");
                fs.tf = find_file(*cx.files, fs.name + ".tf");
                if (fs.tf) {
                    std::lock_guard<std::mutex> lk(*cx.names_mu);
                    const std::string fname = fs.name + ".tf";
                    for (size_t k = 0; k < cx.file_table->size(); ++k)
                        if ((*cx.file_table)[k] == fname) fs.file_id = static_cast<int>(k);
                    if (fs.file_id < 0 && cx.file_table->size() < 255) {
                        cx.file_table->push_back(fname);
                        fs.file_id = static_cast<int>(cx.file_table->size() - 1);
                    }
                }
                cx.fam_cache.push_back(std::move(fs));
            }
            fams[i].slot = slot;
            fams[i].off = c.varu();
            fams[i].size = c.varu();
        }
        // fields: columnFamilyMetadata.unmarshal, column_metadata.go:108-122
        uint64_t nf = c.varu();
        for (uint64_t i = 0; i < nf && !c.bad; ++i) {
            DevCol col{};
            uint64_t nl = c.varu();
            if (c.bad || c.left() < nl) {
                c.bad = true;
                break;
            }
            const uint8_t *np = c.p;
            c.p += nl;
            col.value_type = c.u8();
            col.off = c.varu();
            uint64_t size = c.varu();
            if (c.bad || size > 0xffffffffu || !in_file(col.off, size, cx.fvf->len)) {
                err = "corrupt field columnMetadata";
                return BYDB_EINVAL;
            }
            col.size = static_cast<uint32_t>(size);
            col.name_id = resolve_name(cx, cx.field_cache, i, "f:", SIZE_MAX, std::string(), np, nl);
            col.file_id = 1;
            cols.push_back(col);
        }
        if (c.bad) {
            err = "corrupt blockMetadata";
            return BYDB_EINVAL;
        }
        size_t tag_pos = 0;
        for (uint64_t fi = 0; fi < nfam; ++fi) {
            const ParseCtx::FamSlot &fs = cx.fam_cache[fams[fi].slot];
            if (!fs.tfm || !fs.tf || fs.file_id < 0 || !in_file(fams[fi].off, fams[fi].size, fs.tfm->len)) {
                err = "tag family '" + fs.name + "': missing or truncated .tf/.tfm";
                return BYDB_EINVAL;
            }
            Cur t{fs.tfm->data + fams[fi].off, fs.tfm->data + fams[fi].off + fams[fi].size};
            uint64_t nc = t.varu();
            for (uint64_t i = 0; i < nc && !t.bad; ++i, ++tag_pos) {
                DevCol col{};
                uint64_t nl = t.varu();
                if (t.bad || t.left() < nl) {
                    t.bad = true;
                    break;
                }
                const uint8_t *np = t.p;
                t.p += nl;
                col.value_type = t.u8();
                col.off = t.varu();
                uint64_t size = t.varu();
                if (t.bad || size > 0xffffffffu || !in_file(col.off, size, fs.tf->len)) {
                    err = "corrupt tag columnMetadata";
                    return BYDB_EINVAL;
                }
                col.size = static_cast<uint32_t>(size);
                col.name_id = resolve_name(cx, cx.tag_cache, tag_pos, "t:", fams[fi].slot, fs.name, np, nl);
                col.file_id = static_cast<uint8_t>(fs.file_id);
                cols.push_back(col);
            }
            if (t.bad) {
                err = "corrupt columnFamilyMetadata";
                return BYDB_EINVAL;
            }
        }
        size_t ncols = cols.size() - b.col_begin;
        if (ncols > 0xffff) {
            err = "too many columns in a block";
            return BYDB_EINVAL;
        }
        b.n_cols = static_cast<uint16_t>(ncols);
        blocks.push_back(b);
    }
    return 0;
}
}  // namespace

int build_part_dir(const std::vector<FileImage> &files, NameTable &names, PartDir &out, std::string &err, size_t batch, size_t n_batches) {
    const FileImage *meta = find_file(files, "meta.bin");
    const FileImage *primary = find_file(files, "primary.bin");
    const FileImage *tsf = find_file(files, "timestamps.bin");
    const FileImage *fvf = find_file(files, "fv.bin");
    if (!meta || !primary || !tsf || !fvf) {
        err = "part needs meta.bin, primary.bin, timestamps.bin and fv.bin";
        return BYDB_ENOENT;
    }
    out.files = {"timestamps.bin", "fv.bin"};
    // meta.bin = zstd(concat primaryBlockMetadata), 40 B records (primary_metadata.go:60-83)
    std::vector<uint8_t> raw;
    int rc = zstd_decompress(meta->data, meta->len, raw, err);
    if (rc) return rc;
    if (raw.size() % 40 != 0) {
        err = "meta.bin: length is not a multiple of 40";
        return BYDB_EINVAL;
    }
    struct Pbm {
        uint64_t sid;
        int64_t mn, mx;
        uint64_t off, size;
    };
    std::vector<Pbm> pbms(raw.size() / 40);
    {
        Cur c{raw.data(), raw.data() + raw.size()};
        for (auto &p : pbms) {
            p.sid = c.u64be();
            p.mn = static_cast<int64_t>(c.u64be());
            p.mx = static_cast<int64_t>(c.u64be());
            p.off = c.u64be();
            p.size = c.u64be();
            if (!in_file(p.off, p.size, primary->len)) {
                err = "primary block outside primary.bin";
                return BYDB_EINVAL;
            }
        }
        for (size_t i = 1; i < pbms.size(); ++i)
            if (pbms[i].sid < pbms[i - 1].sid) {  // primary_metadata.go:127-134
                err = "primaryBlockMetadata out of order";
                return BYDB_EINVAL;
            }
    }
    // primary blocks are independent zstd frames: decompress + parse them on a few threads
    if (n_batches > 1) {
        const size_t all = pbms.size();
        const size_t a = all * batch / n_batches, b = all * (batch + 1) / n_batches;
        pbms = std::vector<Pbm>(pbms.begin() + static_cast<long>(a), pbms.begin() + static_cast<long>(b));
    }
    const size_t np = pbms.size();
    unsigned hw = std::thread::hardware_concurrency();
    const size_t nt = std::max<size_t>(1, std::min<size_t>({np, hw ? hw : 4, size_t{16}}));
    std::vector<std::vector<DevBlock>> tb(nt);
    std::vector<std::vector<DevCol>> tc(nt);
    std::vector<int> trc(nt, 0);
    std::vector<std::string> terr(nt);
    std::mutex names_mu;
    auto work = [&](size_t t) {
      try {
        ParseCtx cx;
        cx.files = &files;
        cx.tsf = tsf;
        cx.fvf = fvf;
        cx.names = &names;
        cx.names_mu = &names_mu;
        cx.file_table = &out.files;
        std::vector<uint8_t> blk;
        for (size_t i = np * t / nt; i < np * (t + 1) / nt && trc[t] == 0; ++i) {
            trc[t] = zstd_decompress(primary->data + pbms[i].off, static_cast<size_t>(pbms[i].size), blk, terr[t]);
            if (trc[t] == 0) trc[t] = parse_primary_block(cx, blk.data(), blk.size(), tb[t], tc[t], terr[t]);
        }
      } catch (const std::exception &e) {  // bad_alloc / length_error on a hostile part: an error code, never std::terminate
        trc[t] = BYDB_ENOMEM;
        terr[t] = std::string("block index: ") + e.what();
      }
    };
    if (nt == 1) {
        work(0);
    } else {
        std::vector<std::thread> th;
        for (size_t t = 0; t < nt; ++t) th.emplace_back(work, t);
        for (auto &x : th) x.join();
    }
    for (size_t t = 0; t < nt; ++t)
        if (trc[t]) {
            err = terr[t];
            return trc[t];
        }
    out.blocks.clear();
    out.cols.clear();
    out.total_rows = 0;
    out.max_block_rows = 0;
    out.min_ts = INT64_MAX;
    out.max_ts = INT64_MIN;
    size_t nb = 0, nc = 0;
    for (size_t t = 0; t < nt; ++t) {
        nb += tb[t].size();
        nc += tc[t].size();
    }
    out.blocks.reserve(nb);
    out.cols.reserve(nc);
    for (size_t t = 0; t < nt; ++t) {
        const uint32_t shift = static_cast<uint32_t>(out.cols.size());
        for (DevBlock b : tb[t]) {
            b.col_begin += shift;
            // block_metadata.go:323-336 validateBlockMetadataOrder (also across primary blocks)
            if (!out.blocks.empty()) {
                const DevBlock &pre = out.blocks.back();
                if (b.sid < pre.sid || (b.sid == pre.sid && b.ts_min < pre.ts_min)) {
                    err = "blockMetadata out of order";
                    return BYDB_EINVAL;
                }
            }
            out.total_rows += b.count;
            out.max_block_rows = std::max(out.max_block_rows, b.count);
            out.min_ts = std::min(out.min_ts, b.ts_min);
            out.max_ts = std::max(out.max_ts, b.ts_max);
            out.blocks.push_back(b);
        }
        out.cols.insert(out.cols.end(), tc[t].begin(), tc[t].end());
    }
    return 0;
}

int count_primary_blocks(const std::vector<FileImage> &files, size_t *n, std::string &err) {
    const FileImage *meta = find_file(files, "meta.bin");
    if (!meta) {
        err = "part needs meta.bin";
        return BYDB_ENOENT;
    }
    std::vector<uint8_t> raw;
    int rc = zstd_decompress(meta->data, meta->len, raw, err);
    if (rc) return rc;
    if (raw.size() % 40 != 0) {
        err = "meta.bin: length is not a multiple of 40";
        return BYDB_EINVAL;
    }
    *n = raw.size() / 40;
    return 0;
}

int merge_part_dirs(std::vector<PartDir> &pieces, PartDir &out, std::string &err) {
    out = PartDir();
    out.files = {"timestamps.bin", "fv.bin"};
    out.min_ts = INT64_MAX;
    out.max_ts = INT64_MIN;
    size_t nb = 0, nc = 0;
    for (const auto &p : pieces) {
        nb += p.blocks.size();
        nc += p.cols.size();
    }
    out.blocks.reserve(nb);
    out.cols.reserve(nc);
    for (auto &p : pieces) {
        // file tables are built in discovery order per piece: map this piece's ids onto the merged table
        std::vector<uint8_t> remap(p.files.size(), 0);
        for (size_t i = 0; i < p.files.size(); ++i) {
            size_t k = 0;
            while (k < out.files.size() && out.files[k] != p.files[i]) ++k;
            if (k == out.files.size()) {
                if (out.files.size() >= 255) {
                    err = "too many tag family files";
                    return BYDB_EINVAL;
                }
                out.files.push_back(p.files[i]);
            }
            remap[i] = static_cast<uint8_t>(k);
        }
        const uint32_t shift = static_cast<uint32_t>(out.cols.size());
        for (DevBlock b : p.blocks) {
            b.col_begin += shift;
            if (!out.blocks.empty()) {
                const DevBlock &pre = out.blocks.back();
                if (b.sid < pre.sid || (b.sid == pre.sid && b.ts_min < pre.ts_min)) {
                    err = "blockMetadata out of order";
                    return BYDB_EINVAL;
                }
            }
            out.blocks.push_back(b);
        }
        for (DevCol c : p.cols) {
            c.file_id = c.file_id < remap.size() ? remap[c.file_id] : 0;
            out.cols.push_back(c);
        }
        out.total_rows += p.total_rows;
        out.max_block_rows = std::max(out.max_block_rows, p.max_block_rows);
        if (!p.blocks.empty()) {
            out.min_ts = std::min(out.min_ts, p.min_ts);
            out.max_ts = std::max(out.max_ts, p.max_ts);
        }
    }
    if (out.blocks.empty()) {
        out.min_ts = 0;
        out.max_ts = 0;
    }
    return 0;
}

}  // namespace bydb
