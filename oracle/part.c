/*
 * part.c -- ORACLE (test infrastructure): measure part writer + reader.
 * Restates banyand/measure/{column.go,block.go,block_metadata.go,column_metadata.go,
 * primary_metadata.go,part.go:162-233,block_writer.go,datapoints.go:190-214}.
 */
#include "oracle_internal.h"

#include <stdio.h>
#include <stdlib.h>
#include <string.h>

static __thread char g_err[512];
const char *ob_last_error(void) { return g_err; }
void ob_set_error(const char *msg) { snprintf(g_err, sizeof g_err, "%s", msg); }

/* =================================================================== column pages (column.go) */
/* column.go:222-234 encodeDefault */
static void encode_default(ob_buf *dst, const ob_bytes *cells, size_t n) {
    ob_buf body = {0};
    if (ob_dictionary_encode(&body, cells, n)) {
        ob_buf_put(dst, OB_ENC_DICTIONARY);
        ob_buf_append(dst, body.p, body.len);
    } else {
        ob_buf_reset(&body);
        ob_bytes_block_encode(&body, cells, n);
        ob_buf_put(dst, OB_ENC_PLAIN);
        ob_buf_append(dst, body.p, body.len);
    }
    ob_buf_free(&body);
}

static int cell_is_null(const ob_bytes *c) { return c->len < 0 || (c->len == 4 && memcmp(c->p, "null", 4) == 0); }

/* column.go:113-220 mustWriteTo / encodeInt64Column / encodeFloat64Column */
void ob_column_encode(ob_buf *dst, int value_type, const ob_bytes *cells, size_t n) {
    if (value_type != OB_VT_INT64 && value_type != OB_VT_FLOAT64) {
        encode_default(dst, cells, n);
        return;
    }
    for (size_t i = 0; i < n; i++) {
        if (cell_is_null(&cells[i])) { /* column.go:147-153, 192-195: Plain marker + default page */
            ob_buf_put(dst, OB_ENC_PLAIN);
            encode_default(dst, cells, n);
            return;
        }
    }
    int64_t *ints = (int64_t *)calloc(n ? n : 1, sizeof(int64_t));
    int16_t exp = 0;
    if (value_type == OB_VT_INT64) {
        for (size_t i = 0; i < n; i++) ints[i] = ob_conv_bytes_to_int64(cells[i].p);
    } else {
        double *fl = (double *)malloc(sizeof(double) * (n ? n : 1));
        for (size_t i = 0; i < n; i++) {
            uint64_t u = 0;
            for (int k = 0; k < 8; k++) u = (u << 8) | cells[i].p[k];
            memcpy(&fl[i], &u, 8);
        }
        int rc = ob_float64_to_decimal_list(ints, fl, n, &exp);
        free(fl);
        if (rc != 0) { /* column.go:203-208 */
            free(ints);
            ob_buf_put(dst, OB_ENC_PLAIN);
            encode_default(dst, cells, n);
            return;
        }
    }
    ob_buf body = {0};
    int64_t first = 0;
    int enc = ob_int64_list_encode(&body, ints, n, &first);
    free(ints);
    uint8_t fb[8];
    ob_conv_int64_to_bytes(first, fb);
    ob_buf_put(dst, (uint8_t)enc);
    if (value_type == OB_VT_FLOAT64) {
        ob_buf_put(dst, (uint8_t)((uint16_t)exp >> 8));
        ob_buf_put(dst, (uint8_t)((uint16_t)exp & 0xff));
    }
    ob_buf_append(dst, fb, 8);
    ob_buf_append(dst, body.p, body.len);
    ob_buf_free(&body);
}

/* column.go:366-379 decodeDefault */
static int decode_default(ob_bytes *out, size_t n, const uint8_t *src, size_t srclen, ob_buf *arena) {
    if (srclen < 1) return -1;
    if (src[0] == OB_ENC_DICTIONARY) return ob_dictionary_decode(out, n, src + 1, srclen - 1, arena);
    return ob_bytes_block_decode(out, n, src + 1, srclen - 1, arena, 0) < 0 ? -1 : 0;
}

/* column.go:276-364 decodeColumnValues / decodeInt64Column / decodeFloat64Column.
 * Numeric cells are re-materialised as 8-byte cells exactly like the reference. */
int ob_column_decode(ob_bytes *out, size_t n, int value_type, const uint8_t *src, size_t srclen, ob_buf *arena) {
    if (value_type != OB_VT_INT64 && value_type != OB_VT_FLOAT64) return decode_default(out, n, src, srclen, arena);
    if (srclen < 1) return -1;
    int enc = src[0];
    if (enc == OB_ENC_PLAIN) return decode_default(out, n, src + 1, srclen - 1, arena);
    int64_t *ints = (int64_t *)malloc(sizeof(int64_t) * (n ? n : 1));
    size_t hdr = value_type == OB_VT_INT64 ? 9 : 11;
    if (srclen < hdr) {
        free(ints);
        return -1;
    }
    int16_t exp = 0;
    if (value_type == OB_VT_FLOAT64) exp = (int16_t)(((uint16_t)src[1] << 8) | src[2]);
    int64_t first = ob_conv_bytes_to_int64(src + hdr - 8);
    if (ob_int64_list_decode(ints, src + hdr, srclen - hdr, enc, first, n) != 0) {
        free(ints);
        return -1;
    }
    /* reserve so pointers stay valid */
    size_t base = arena->len;
    for (size_t i = 0; i < n; i++) {
        uint8_t cell[8];
        if (value_type == OB_VT_INT64) {
            ob_conv_int64_to_bytes(ints[i], cell);
        } else {
            double f;
            ob_decimal_list_to_float64(&f, &ints[i], 1, exp);
            uint64_t u;
            memcpy(&u, &f, 8);
            for (int k = 0; k < 8; k++) cell[k] = (uint8_t)(u >> (56 - 8 * k));
        }
        ob_buf_append(arena, cell, 8);
    }
    for (size_t i = 0; i < n; i++) {
        out[i].p = arena->p + base + 8 * i;
        out[i].len = 8;
    }
    free(ints);
    return 0;
}

/* =================================================================== metadata marshal */
static void put_u64be(ob_buf *b, uint64_t u) {
    for (int k = 7; k >= 0; k--) ob_buf_put(b, (uint8_t)(u >> (8 * k)));
}
static uint64_t get_u64be(const uint8_t *p) {
    uint64_t u = 0;
    for (int k = 0; k < 8; k++) u = (u << 8) | p[k];
    return u;
}
/* bytes.go:28-32 EncodeBytes */
static void put_bytes(ob_buf *b, const char *s) {
    size_t n = strlen(s);
    ob_varuint64_append(b, n);
    ob_buf_append(b, s, n);
}

/* column_metadata.go:47-52 + :99-106 */
static void cfm_marshal(ob_buf *dst, const obi_colmeta *cms, size_t n) {
    ob_varuint64_append(dst, n);
    for (size_t i = 0; i < n; i++) {
        put_bytes(dst, cms[i].name);
        ob_buf_put(dst, (uint8_t)cms[i].value_type);
        ob_varuint64_append(dst, cms[i].offset);
        ob_varuint64_append(dst, cms[i].size);
    }
}

/* reads a varuint the way the reference does (failure -> value 0, nothing consumed) */
static const uint8_t *rd_varu(const uint8_t *p, const uint8_t *end, uint64_t *out) {
    size_t used = ob_varuint64_read(p, (size_t)(end - p), out);
    return p + used;
}

/* column_metadata.go:54-67, :108-122; returns new cursor or NULL */
const uint8_t *obi_cfm_unmarshal(const uint8_t *p, const uint8_t *end, obi_colmeta **out, size_t *n_out) {
    uint64_t n;
    p = rd_varu(p, end, &n);
    *out = NULL;
    *n_out = 0;
    if (n < 1) return p;
    obi_colmeta *cms = (obi_colmeta *)calloc((size_t)n, sizeof(obi_colmeta));
    for (uint64_t i = 0; i < n; i++) {
        uint64_t nl;
        p = rd_varu(p, end, &nl);
        if ((uint64_t)(end - p) < nl || nl >= sizeof(cms[i].name)) {
            free(cms);
            return NULL;
        }
        memcpy(cms[i].name, p, (size_t)nl);
        cms[i].name[nl] = 0;
        p += nl;
        if (p >= end) {
            free(cms);
            return NULL;
        }
        cms[i].value_type = *p++;
        p = rd_varu(p, end, &cms[i].offset);
        p = rd_varu(p, end, &cms[i].size);
    }
    *out = cms;
    *n_out = (size_t)n;
    return p;
}

/* block_metadata.go:113-131 marshal (+ timestampsMetadata :268-277) */
static void bm_marshal(ob_buf *dst, const obi_blockmeta *bm) {
    put_u64be(dst, bm->sid);
    ob_varuint64_append(dst, bm->uncompressed);
    ob_varuint64_append(dst, bm->count);
    ob_varuint64_append(dst, bm->ts_off);
    ob_varuint64_append(dst, bm->ts_size);
    put_u64be(dst, (uint64_t)bm->ts_min);
    put_u64be(dst, (uint64_t)bm->ts_max);
    ob_buf_put(dst, (uint8_t)bm->ts_enc);
    ob_varuint64_append(dst, bm->ver_off);
    put_u64be(dst, (uint64_t)bm->ver_first);
    ob_buf_put(dst, (uint8_t)bm->ver_enc);
    ob_varuint64_append(dst, bm->n_fams);
    /* sorted by family name (block_metadata.go:119-124); fams[] is kept sorted by the writer */
    for (size_t i = 0; i < bm->n_fams; i++) {
        put_bytes(dst, bm->fams[i].name);
        ob_varuint64_append(dst, bm->fams[i].offset);
        ob_varuint64_append(dst, bm->fams[i].size);
    }
    cfm_marshal(dst, bm->fields, bm->n_fields);
}

void obi_bm_free(obi_blockmeta *bm) {
    free(bm->fams);
    free(bm->fields);
    bm->fams = NULL;
    bm->fields = NULL;
}

/* block_metadata.go:133-168 unmarshal (+ :279-293) */
const uint8_t *obi_bm_unmarshal(const uint8_t *p, const uint8_t *end, obi_blockmeta *bm) {
    memset(bm, 0, sizeof *bm);
    if (end - p < 8) return NULL;
    bm->sid = get_u64be(p);
    p += 8;
    p = rd_varu(p, end, &bm->uncompressed);
    p = rd_varu(p, end, &bm->count);
    p = rd_varu(p, end, &bm->ts_off);
    p = rd_varu(p, end, &bm->ts_size);
    if (end - p < 17) return NULL;
    bm->ts_min = (int64_t)get_u64be(p);
    p += 8;
    bm->ts_max = (int64_t)get_u64be(p);
    p += 8;
    bm->ts_enc = *p++;
    p = rd_varu(p, end, &bm->ver_off);
    if (end - p < 9) return NULL;
    bm->ver_first = (int64_t)get_u64be(p);
    p += 8;
    bm->ver_enc = *p++;
    uint64_t nf;
    p = rd_varu(p, end, &nf);
    if (nf > 0) {
        bm->fams = (obi_fammeta *)calloc((size_t)nf, sizeof(obi_fammeta));
        bm->n_fams = (size_t)nf;
        for (uint64_t i = 0; i < nf; i++) {
            uint64_t nl;
            p = rd_varu(p, end, &nl);
            if ((uint64_t)(end - p) < nl || nl >= sizeof(bm->fams[i].name)) {
                obi_bm_free(bm);
                return NULL;
            }
            memcpy(bm->fams[i].name, p, (size_t)nl);
            bm->fams[i].name[nl] = 0;
            p += nl;
            p = rd_varu(p, end, &bm->fams[i].offset);
            p = rd_varu(p, end, &bm->fams[i].size);
        }
    }
    p = obi_cfm_unmarshal(p, end, &bm->fields, &bm->n_fields);
    if (!p) {
        obi_bm_free(bm);
        return NULL;
    }
    return p;
}

/* =================================================================== part container */
obi_file *obi_part_file(ob_part *p, const char *name, int create) {
    for (int i = 0; i < p->n_files; i++)
        if (strcmp(p->files[i]->name, name) == 0) return p->files[i];
    if (!create) return NULL;
    p->files = (obi_file **)realloc(p->files, sizeof(obi_file *) * (size_t)(p->n_files + 1));
    obi_file *f = (obi_file *)calloc(1, sizeof(obi_file)); /* stable address: callers keep pointers */
    p->files[p->n_files++] = f;
    snprintf(f->name, sizeof f->name, "%s", name);
    return f;
}
int ob_part_n_files(const ob_part *p) { return p->n_files; }
const char *ob_part_file_name(const ob_part *p, int i) { return p->files[i]->name; }
const uint8_t *ob_part_file_data(const ob_part *p, int i, size_t *len) {
    *len = p->files[i]->data.len;
    return p->files[i]->data.p;
}
void ob_part_meta(const ob_part *p, uint64_t *total_count, uint64_t *blocks_count, int64_t *min_ts, int64_t *max_ts,
                  uint64_t *uncompressed, uint64_t *compressed) {
    if (total_count) *total_count = p->total_count;
    if (blocks_count) *blocks_count = p->blocks_count;
    if (min_ts) *min_ts = p->min_ts;
    if (max_ts) *max_ts = p->max_ts;
    if (uncompressed) *uncompressed = p->uncompressed;
    if (compressed) *compressed = p->compressed;
}
void ob_part_free(ob_part *p) {
    if (!p) return;
    for (int i = 0; i < p->n_files; i++) {
        ob_buf_free(&p->files[i]->data);
        free(p->files[i]);
    }
    free(p->files);
    free(p->pbm);
    free(p);
}

/* primary_metadata.go:106-134 unmarshalPrimaryBlockMetadata (meta.bin is one zstd frame, :84-104) */
static int part_load_primary_index(ob_part *p) {
    obi_file *meta = obi_part_file(p, "meta.bin", 0);
    if (!meta) {
        ob_set_error("part has no meta.bin");
        return -1;
    }
    ob_buf raw = {0};
    if (ob_zstd_decompress(&raw, meta->data.p, meta->data.len) != 0) {
        ob_set_error("cannot decompress meta.bin");
        return -1;
    }
    if (raw.len % 40 != 0) {
        ob_buf_free(&raw);
        ob_set_error("meta.bin: size not a multiple of 40");
        return -1;
    }
    p->n_pbm = raw.len / 40;
    p->pbm = (obi_primary *)calloc(p->n_pbm ? p->n_pbm : 1, sizeof(obi_primary));
    for (size_t i = 0; i < p->n_pbm; i++) {
        const uint8_t *s = raw.p + 40 * i;
        p->pbm[i].sid = get_u64be(s);
        p->pbm[i].min_ts = (int64_t)get_u64be(s + 8);
        p->pbm[i].max_ts = (int64_t)get_u64be(s + 16);
        p->pbm[i].offset = get_u64be(s + 24);
        p->pbm[i].size = get_u64be(s + 32);
        if (i > 0 && p->pbm[i].sid < p->pbm[i - 1].sid) { /* :127-134 */
            ob_buf_free(&raw);
            ob_set_error("primaryBlockMetadata out of order");
            return -1;
        }
    }
    ob_buf_free(&raw);
    return 0;
}

/* part.go:312-375 mustOpenFilePart (from in-memory file images) */
ob_part *ob_part_open(int n_files, const char *const *names, const uint8_t *const *data, const size_t *lens) {
    ob_part *p = (ob_part *)calloc(1, sizeof *p);
    for (int i = 0; i < n_files; i++) {
        obi_file *f = obi_part_file(p, names[i], 1);
        ob_buf_append(&f->data, data[i], lens[i]);
    }
    if (part_load_primary_index(p) != 0) {
        ob_part_free(p);
        return NULL;
    }
    /* metadata.json is not needed by the scan; recompute the counters from the block index */
    obi_blockmeta *bms;
    size_t nb;
    p->min_ts = INT64_MAX;
    p->max_ts = INT64_MIN;
    for (size_t i = 0; i < p->n_pbm; i++) {
        if (obi_part_read_primary_block(p, i, &bms, &nb) != 0) {
            ob_part_free(p);
            return NULL;
        }
        for (size_t k = 0; k < nb; k++) {
            p->total_count += bms[k].count;
            p->uncompressed += bms[k].uncompressed;
            if (bms[k].ts_min < p->min_ts) p->min_ts = bms[k].ts_min;
            if (bms[k].ts_max > p->max_ts) p->max_ts = bms[k].ts_max;
            obi_bm_free(&bms[k]);
        }
        p->blocks_count += nb;
        free(bms);
    }
    for (int i = 0; i < p->n_files; i++) p->compressed += p->files[i]->data.len;
    return p;
}

/* part_iter.go:184-208 readPrimaryBlock: zstd-decompress one primary block, unmarshal blockMetadata[] */
int obi_part_read_primary_block(ob_part *p, size_t idx, obi_blockmeta **out, size_t *n_out) {
    obi_file *pf = obi_part_file(p, "primary.bin", 0);
    if (!pf || idx >= p->n_pbm) return -1;
    const obi_primary *pb = &p->pbm[idx];
    if (pb->offset + pb->size > pf->data.len) {
        ob_set_error("primary block out of file bounds");
        return -1;
    }
    ob_buf raw = {0};
    if (ob_zstd_decompress(&raw, pf->data.p + pb->offset, (size_t)pb->size) != 0) {
        ob_set_error("cannot decompress primary block");
        return -1;
    }
    size_t cap = 64, n = 0;
    obi_blockmeta *bms = (obi_blockmeta *)malloc(sizeof(obi_blockmeta) * cap);
    const uint8_t *s = raw.p, *end = raw.p + raw.len;
    while (s < end) {
        if (n == cap) {
            cap *= 2;
            bms = (obi_blockmeta *)realloc(bms, sizeof(obi_blockmeta) * cap);
        }
        s = obi_bm_unmarshal(s, end, &bms[n]);
        if (!s) {
            for (size_t k = 0; k < n; k++) obi_bm_free(&bms[k]);
            free(bms);
            ob_buf_free(&raw);
            ob_set_error("cannot unmarshal blockMetadata");
            return -1;
        }
        /* block_metadata.go:323-336 validateBlockMetadataOrder */
        if (n > 0 && (bms[n].sid < bms[n - 1].sid || (bms[n].sid == bms[n - 1].sid && bms[n].ts_min < bms[n - 1].ts_min))) {
            for (size_t k = 0; k <= n; k++) obi_bm_free(&bms[k]);
            free(bms);
            ob_buf_free(&raw);
            ob_set_error("blockMetadata out of order");
            return -1;
        }
        n++;
    }
    ob_buf_free(&raw);
    *out = bms;
    *n_out = n;
    return 0;
}

/* =================================================================== builder */
typedef struct {
    char name[128];
    int value_type;
    /* per-row cell storage: offsets into data (-1 = nil) */
    int64_t *off;
    int32_t *len;
    ob_buf data;
} bcol;
typedef struct {
    char name[128];
    int n_cols;
    bcol *cols;
} bfam;

struct ob_builder {
    size_t n, cap;
    uint64_t *sids;
    int64_t *ts, *ver;
    int n_fields;
    bcol *fields;
    int n_fams;
    bfam *fams;
    int schema_set;
};

ob_builder *ob_builder_new(void) { return (ob_builder *)calloc(1, sizeof(ob_builder)); }

static void bcol_free(bcol *c) {
    free(c->off);
    free(c->len);
    ob_buf_free(&c->data);
}
void ob_builder_free(ob_builder *b) {
    if (!b) return;
    for (int i = 0; i < b->n_fields; i++) bcol_free(&b->fields[i]);
    free(b->fields);
    for (int i = 0; i < b->n_fams; i++) {
        for (int j = 0; j < b->fams[i].n_cols; j++) bcol_free(&b->fams[i].cols[j]);
        free(b->fams[i].cols);
    }
    free(b->fams);
    free(b->sids);
    free(b->ts);
    free(b->ver);
    free(b);
}

static void bcol_init(bcol *c, const ob_column *src) {
    memset(c, 0, sizeof *c);
    snprintf(c->name, sizeof c->name, "%s", src->name);
    c->value_type = src->value_type;
}
static void bcol_append(bcol *c, const ob_column *src, size_t base, size_t n, size_t newcap) {
    c->off = (int64_t *)realloc(c->off, sizeof(int64_t) * newcap);
    c->len = (int32_t *)realloc(c->len, sizeof(int32_t) * newcap);
    for (size_t i = 0; i < n; i++) {
        size_t r = base + i;
        if (src->value_type == OB_VT_INT64 || src->value_type == OB_VT_FLOAT64) {
            if (src->nulls && src->nulls[i]) {
                c->off[r] = -1;
                c->len[r] = -1;
                continue;
            }
            uint8_t cell[8];
            if (src->value_type == OB_VT_INT64) {
                ob_conv_int64_to_bytes(src->i64[i], cell); /* write_standalone.go:520-523 */
            } else {
                uint64_t u;
                memcpy(&u, &src->f64[i], 8); /* write_standalone.go:525-528, number.go:128-132 */
                for (int k = 0; k < 8; k++) cell[k] = (uint8_t)(u >> (56 - 8 * k));
            }
            c->off[r] = (int64_t)c->data.len;
            c->len[r] = 8;
            ob_buf_append(&c->data, cell, 8);
        } else {
            if (src->bytes[i].len < 0) {
                c->off[r] = -1;
                c->len[r] = -1;
                continue;
            }
            c->off[r] = (int64_t)c->data.len;
            c->len[r] = (int32_t)src->bytes[i].len;
            ob_buf_append(&c->data, src->bytes[i].p, (size_t)src->bytes[i].len);
        }
    }
}

int ob_builder_append(ob_builder *b, size_t n, const uint64_t *sids, const int64_t *ts, const int64_t *versions,
                      int n_fields, const ob_column *fields, int n_fams, const ob_family *fams) {
    if (!b->schema_set) {
        b->n_fields = n_fields;
        b->fields = (bcol *)calloc((size_t)(n_fields ? n_fields : 1), sizeof(bcol));
        for (int i = 0; i < n_fields; i++) bcol_init(&b->fields[i], &fields[i]);
        b->n_fams = n_fams;
        b->fams = (bfam *)calloc((size_t)(n_fams ? n_fams : 1), sizeof(bfam));
        for (int i = 0; i < n_fams; i++) {
            snprintf(b->fams[i].name, sizeof b->fams[i].name, "%s", fams[i].name);
            b->fams[i].n_cols = fams[i].n_cols;
            b->fams[i].cols = (bcol *)calloc((size_t)(fams[i].n_cols ? fams[i].n_cols : 1), sizeof(bcol));
            for (int j = 0; j < fams[i].n_cols; j++) bcol_init(&b->fams[i].cols[j], &fams[i].cols[j]);
        }
        b->schema_set = 1;
    } else if (n_fields != b->n_fields || n_fams != b->n_fams) {
        ob_set_error("builder: schema mismatch");
        return -1;
    }
    size_t newcap = b->n + n;
    b->sids = (uint64_t *)realloc(b->sids, sizeof(uint64_t) * (newcap ? newcap : 1));
    b->ts = (int64_t *)realloc(b->ts, sizeof(int64_t) * (newcap ? newcap : 1));
    b->ver = (int64_t *)realloc(b->ver, sizeof(int64_t) * (newcap ? newcap : 1));
    memcpy(b->sids + b->n, sids, sizeof(uint64_t) * n);
    memcpy(b->ts + b->n, ts, sizeof(int64_t) * n);
    memcpy(b->ver + b->n, versions, sizeof(int64_t) * n);
    for (int i = 0; i < n_fields; i++) bcol_append(&b->fields[i], &fields[i], b->n, n, newcap ? newcap : 1);
    for (int i = 0; i < n_fams; i++)
        for (int j = 0; j < fams[i].n_cols; j++) bcol_append(&b->fams[i].cols[j], &fams[i].cols[j], b->n, n, newcap ? newcap : 1);
    b->n = newcap;
    return 0;
}

/* sort context (datapoints.go:190-198 Less: sid asc, ts asc, version desc) */
static __thread const ob_builder *g_sort_b;
static int row_cmp(const void *pa, const void *pb) {
    size_t a = *(const size_t *)pa, c = *(const size_t *)pb;
    const ob_builder *b = g_sort_b;
    if (b->sids[a] != b->sids[c]) return b->sids[a] < b->sids[c] ? -1 : 1;
    if (b->ts[a] != b->ts[c]) return b->ts[a] < b->ts[c] ? -1 : 1;
    if (b->ver[a] != b->ver[c]) return b->ver[a] > b->ver[c] ? -1 : 1;
    return a < c ? -1 : (a > c ? 1 : 0); /* stable tiebreak; the reference's sort.Sort is unstable here */
}

static size_t cell_size(const bcol *c, size_t r) { return c->len[r] > 0 ? (size_t)c->len[r] : 0; }

/* part.go:234-249 uncompressedDataPointSizeBytes. The field family (nameValues) name is "" in the
 * writer used by the reference tests; tag family names count once per family per row. */
static uint64_t row_uncompressed(const ob_builder *b, size_t r) {
    uint64_t n = 16;
    for (int i = 0; i < b->n_fields; i++) n += strlen(b->fields[i].name) + cell_size(&b->fields[i], r);
    for (int i = 0; i < b->n_fams; i++) {
        n += strlen(b->fams[i].name);
        for (int j = 0; j < b->fams[i].n_cols; j++) n += strlen(b->fams[i].cols[j].name) + cell_size(&b->fams[i].cols[j], r);
    }
    return n;
}

typedef struct {
    ob_part *part;
    ob_buf primary_block; /* bw.primaryBlockData */
    ob_buf meta_data;     /* bw.metaData */
    uint64_t sid_first, sid_last;
    int64_t min_ts, max_ts, min_ts_last;
    int has_written;
} bwriter;

static void cells_of(const bcol *c, const size_t *rows, size_t n, ob_bytes *cells) {
    for (size_t i = 0; i < n; i++) {
        size_t r = rows[i];
        if (c->len[r] < 0) {
            cells[i].p = NULL;
            cells[i].len = -1;
        } else {
            cells[i].p = c->data.p + c->off[r];
            cells[i].len = c->len[r];
        }
    }
}

/* block_writer.go:247-262 mustFlushPrimaryBlock + primary_metadata.go:47-58 mustWriteBlock */
static void flush_primary(bwriter *w) {
    if (w->primary_block.len > 0) {
        obi_file *pf = obi_part_file(w->part, "primary.bin", 1);
        uint64_t off = pf->data.len;
        ob_zstd_compress(&pf->data, w->primary_block.p, w->primary_block.len, 1);
        uint64_t size = pf->data.len - off;
        put_u64be(&w->meta_data, w->sid_first);
        put_u64be(&w->meta_data, (uint64_t)w->min_ts);
        put_u64be(&w->meta_data, (uint64_t)w->max_ts);
        put_u64be(&w->meta_data, off);
        put_u64be(&w->meta_data, size);
    }
    w->has_written = 0;
    w->min_ts = w->max_ts = 0;
    w->sid_first = 0;
    ob_buf_reset(&w->primary_block);
}

static int fam_name_cmp(const void *a, const void *b) { return strcmp(((const obi_fammeta *)a)->name, ((const obi_fammeta *)b)->name); }

/* block_writer.go:206-245 mustWriteBlock + block.go:139-160 mustWriteTo */
static void write_block(bwriter *w, const ob_builder *b, uint64_t sid, const size_t *rows, size_t n) {
    if (n == 0) return;
    ob_part *p = w->part;
    obi_blockmeta bm;
    memset(&bm, 0, sizeof bm);
    bm.sid = sid;
    bm.count = n;
    /* block.go:267-297 uncompressedSizeBytes */
    uint64_t unc = (uint64_t)n * 16;
    for (int i = 0; i < b->n_fams; i++) {
        unc += strlen(b->fams[i].name);
        for (int j = 0; j < b->fams[i].n_cols; j++) {
            unc += strlen(b->fams[i].cols[j].name);
            for (size_t k = 0; k < n; k++) unc += cell_size(&b->fams[i].cols[j], rows[k]);
        }
    }
    for (int i = 0; i < b->n_fields; i++) {
        size_t nl = strlen(b->fields[i].name);
        for (size_t k = 0; k < n; k++) {
            size_t cs = cell_size(&b->fields[i], rows[k]);
            if (cs > 0) unc += nl + cs;
        }
    }
    bm.uncompressed = unc;

    /* block.go:361-379 mustWriteTimestampsTo */
    int64_t *tmp = (int64_t *)malloc(sizeof(int64_t) * n);
    obi_file *tsf = obi_part_file(p, "timestamps.bin", 1);
    ob_buf body = {0};
    for (size_t k = 0; k < n; k++) tmp[k] = b->ts[rows[k]];
    int64_t first = 0;
    int enc = ob_int64_list_encode(&body, tmp, n, &first);
    bm.ts_enc = enc + 4; /* GetVersionType, encoding.go:102-115 */
    bm.ts_min = first;
    bm.ts_max = tmp[n - 1];
    bm.ts_off = tsf->data.len;
    bm.ver_off = body.len;
    ob_buf_append(&tsf->data, body.p, body.len);
    ob_buf_reset(&body);
    for (size_t k = 0; k < n; k++) tmp[k] = b->ver[rows[k]];
    bm.ver_enc = ob_int64_list_encode(&body, tmp, n, &first);
    bm.ver_first = first;
    bm.ts_size = bm.ver_off + body.len;
    ob_buf_append(&tsf->data, body.p, body.len);
    free(tmp);

    ob_bytes *cells = (ob_bytes *)malloc(sizeof(ob_bytes) * n);
    /* tag families: block.go:184-205 marshalTagFamily */
    bm.n_fams = (size_t)b->n_fams;
    bm.fams = (obi_fammeta *)calloc((size_t)(b->n_fams ? b->n_fams : 1), sizeof(obi_fammeta));
    for (int i = 0; i < b->n_fams; i++) {
        char fn[160];
        snprintf(fn, sizeof fn, "%s.tf", b->fams[i].name);
        obi_file *tf = obi_part_file(p, fn, 1);
        snprintf(fn, sizeof fn, "%s.tfm", b->fams[i].name);
        obi_file *tfm = obi_part_file(p, fn, 1);
        int nc = b->fams[i].n_cols;
        obi_colmeta *cms = (obi_colmeta *)calloc((size_t)(nc ? nc : 1), sizeof(obi_colmeta));
        for (int j = 0; j < nc; j++) {
            const bcol *c = &b->fams[i].cols[j];
            cells_of(c, rows, n, cells);
            ob_buf_reset(&body);
            ob_column_encode(&body, c->value_type, cells, n);
            snprintf(cms[j].name, sizeof cms[j].name, "%s", c->name);
            cms[j].value_type = c->value_type;
            cms[j].offset = tf->data.len;
            cms[j].size = body.len;
            ob_buf_append(&tf->data, body.p, body.len);
        }
        ob_buf_reset(&body);
        cfm_marshal(&body, cms, (size_t)nc);
        free(cms);
        snprintf(bm.fams[i].name, sizeof bm.fams[i].name, "%s", b->fams[i].name);
        bm.fams[i].offset = tfm->data.len;
        bm.fams[i].size = body.len;
        ob_buf_append(&tfm->data, body.p, body.len);
    }
    qsort(bm.fams, bm.n_fams, sizeof(obi_fammeta), fam_name_cmp);
    /* fields: block.go:154-159 */
    obi_file *fv = obi_part_file(p, "fv.bin", 1);
    bm.n_fields = (size_t)b->n_fields;
    bm.fields = (obi_colmeta *)calloc((size_t)(b->n_fields ? b->n_fields : 1), sizeof(obi_colmeta));
    for (int i = 0; i < b->n_fields; i++) {
        const bcol *c = &b->fields[i];
        cells_of(c, rows, n, cells);
        ob_buf_reset(&body);
        ob_column_encode(&body, c->value_type, cells, n);
        snprintf(bm.fields[i].name, sizeof bm.fields[i].name, "%s", c->name);
        bm.fields[i].value_type = c->value_type;
        bm.fields[i].offset = fv->data.len;
        bm.fields[i].size = body.len;
        ob_buf_append(&fv->data, body.p, body.len);
    }
    free(cells);
    ob_buf_free(&body);

    /* block_writer.go:213-245 bookkeeping */
    int had = w->has_written;
    if (!had) {
        w->sid_first = sid;
        w->has_written = 1;
    }
    w->sid_last = sid;
    if (p->total_count == 0 || bm.ts_min < p->min_ts) p->min_ts = bm.ts_min;
    if (p->total_count == 0 || bm.ts_max > p->max_ts) p->max_ts = bm.ts_max;
    if (!had || bm.ts_min < w->min_ts) w->min_ts = bm.ts_min;
    if (!had || bm.ts_max > w->max_ts) w->max_ts = bm.ts_max;
    w->min_ts_last = bm.ts_min;
    p->uncompressed += bm.uncompressed;
    p->total_count += bm.count;
    p->blocks_count++;
    bm_marshal(&w->primary_block, &bm);
    obi_bm_free(&bm);
    if (w->primary_block.len > OBI_MAX_UNCOMPRESSED_PRIMARY) flush_primary(w);
}

/* one block of a builder: rows keep[start, start + n) of series sid */
typedef struct {
    uint64_t sid;
    size_t start, n;
} bcut;
typedef struct {
    size_t *keep; /* surviving rows in (sid, ts, -version) order */
    bcut *cuts;
    size_t n_cuts;
} bblocks;

/* part.go:162-205 mustInitFromDataPoints: sort, dedup exactly as part.go:176-190 (note the tsPrev==0 quirk for the very
 * first row) and cut into blocks; a cut of n == 0 is written as nothing, as write_block skips it */
static void cut_blocks(const ob_builder *b, bblocks *out) {
    size_t *perm = (size_t *)malloc(sizeof(size_t) * (b->n ? b->n : 1));
    for (size_t i = 0; i < b->n; i++) perm[i] = i;
    g_sort_b = b;
    qsort(perm, b->n, sizeof(size_t), row_cmp);
    out->keep = (size_t *)malloc(sizeof(size_t) * (b->n ? b->n : 1));
    out->cuts = (bcut *)malloc(sizeof(bcut) * (b->n + 1));
    out->n_cuts = 0;
    size_t m = 0, index_prev = 0;
    uint64_t sid_prev = 0, unc = 0;
    int64_t ts_prev = 0;
    for (size_t i = 0; i < b->n; i++) {
        size_t r = perm[i];
        uint64_t sid = b->sids[r];
        if (sid_prev == 0) sid_prev = sid;
        if (sid == sid_prev) {
            if (ts_prev == b->ts[r]) continue; /* dps.skip(i) */
            ts_prev = b->ts[r];
        }
        /* row survives at position m */
        if (unc >= OBI_MAX_UNCOMPRESSED_BLOCK || (m - index_prev) > OBI_MAX_BLOCK_LENGTH || sid != sid_prev) {
            out->cuts[out->n_cuts++] = (bcut){sid_prev, index_prev, m - index_prev};
            sid_prev = sid;
            index_prev = m;
            ts_prev = b->ts[r];
            unc = 0;
        }
        out->keep[m++] = r;
        unc += row_uncompressed(b, r);
    }
    out->cuts[out->n_cuts++] = (bcut){sid_prev, index_prev, m - index_prev};
    free(perm);
}

/* part.go:162-205 mustInitFromDataPoints + block_writer.go:264-285 Flush */
ob_part *ob_builder_finish(ob_builder *b) { return ob_builder_finish_many(&b, 1); }

/* One part from several builders, each with its own schema: a part holds every series of its group and shard, and each
 * block carries the tag families and fields of its own series (block.go:88-123 processTagFamilies / processTags).  Each
 * builder's rows are cut exactly as ob_builder_finish cuts them; the blocks of all builders then go through one block
 * writer in series order (part.go:192-205, block_writer.go:206-245), so primary blocks mix schemas and the .tf / .tfm
 * files are shared by family name. */
ob_part *ob_builder_finish_many(ob_builder *const *bs, int n_builders) {
    ob_part *p = (ob_part *)calloc(1, sizeof *p);
    /* fixed file order for reproducibility */
    obi_part_file(p, "meta.bin", 1);
    obi_part_file(p, "primary.bin", 1);
    obi_part_file(p, "timestamps.bin", 1);
    obi_part_file(p, "fv.bin", 1);
    size_t total = 0;
    for (int k = 0; k < n_builders; k++) total += bs[k]->n;
    if (total == 0) {
        ob_zstd_compress(&obi_part_file(p, "meta.bin", 0)->data, "", 0, 1);
        return p;
    }
    bblocks *bb = (bblocks *)calloc((size_t)n_builders, sizeof(bblocks));
    size_t *next = (size_t *)calloc((size_t)n_builders, sizeof(size_t));
    for (int k = 0; k < n_builders; k++)
        if (bs[k]->n) cut_blocks(bs[k], &bb[k]);
    bwriter w;
    memset(&w, 0, sizeof w);
    w.part = p;
    int overlap = 0;
    for (;;) {
        /* the builder whose next block has the smallest series; series of different builders never meet */
        int best = -1;
        for (int k = 0; k < n_builders; k++) {
            if (next[k] >= bb[k].n_cuts) continue;
            if (best >= 0 && bb[k].cuts[next[k]].sid == bb[best].cuts[next[best]].sid) overlap = 1;
            if (best < 0 || bb[k].cuts[next[k]].sid < bb[best].cuts[next[best]].sid) best = k;
        }
        if (best < 0 || overlap) break;
        const uint64_t sid = bb[best].cuts[next[best]].sid;
        while (next[best] < bb[best].n_cuts && bb[best].cuts[next[best]].sid == sid) {
            const bcut *c = &bb[best].cuts[next[best]++];
            write_block(&w, bs[best], c->sid, bb[best].keep + c->start, c->n);
        }
    }
    for (int k = 0; k < n_builders; k++) {
        free(bb[k].keep);
        free(bb[k].cuts);
    }
    free(bb);
    free(next);
    if (overlap) {
        ob_buf_free(&w.meta_data);
        ob_buf_free(&w.primary_block);
        ob_part_free(p);
        ob_set_error("builder: a series appears in more than one builder");
        return NULL;
    }
    flush_primary(&w);
    ob_zstd_compress(&obi_part_file(p, "meta.bin", 0)->data, w.meta_data.p, w.meta_data.len, 1);
    ob_buf_free(&w.meta_data);
    ob_buf_free(&w.primary_block);
    for (int i = 0; i < p->n_files; i++) p->compressed += p->files[i]->data.len;
    if (part_load_primary_index(p) != 0) {
        ob_part_free(p);
        return NULL;
    }
    return p;
}
