/*
 * query.c -- ORACLE (test infrastructure): the measure scan -> filter -> aggregate path on the CPU.
 * Restates, in the reference's own structure:
 *   block selection      banyand/measure/part_iter.go:79-250, query.go:594-639
 *   block load + trim    banyand/measure/block.go:299-418, 793-870; pkg/timestamp/range.go:143-169
 *   merge + version dedup banyand/measure/query.go:912-1025, query_batch.go:124-181
 *   fold / finalize      pkg/query/vectorized/measure/aggregation.go:193-334, pkg/query/aggregation/function.go
 *   top                  pkg/query/vectorized/measure/top.go:145-214
 * Row predicates on stored (non-indexed) tag columns are an extension the reference does not have
 * (SURVEY.md F3); they are defined here as a plain per-row filter applied after merge/dedup.
 */
#include "oracle_internal.h"

#include <float.h>
#include <math.h>
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
    int is_float;
    int present;
    int64_t *i64;
    double *f64;
    uint8_t *null; /* NULL = no nulls */
} fcol;

typedef struct {
    int present;
    int value_type;
    ob_bytes *cells;
    ob_buf arena;
} tcol;

typedef struct {
    int part;
    obi_blockmeta bm;
    size_t n; /* rows after time trim */
    int64_t *ts, *ver;
    fcol *fields; /* [n_fcols] */
    tcol *tags;   /* [n_preds] */
    size_t idx;
    int blank;
} cursor;

typedef struct {
    const ob_query *q;
    int n_fcols;
    const char **fcol_names;
    int *agg_fcol; /* agg -> fcol */
    cursor *cur;
    size_t n_cur;
} scan;

static int64_t wadd(int64_t a, int64_t b) { return (int64_t)((uint64_t)a + (uint64_t)b); }

/* ------------------------------------------------------------------ block selection */
static int sid_selected(const ob_query *q, uint64_t sid, size_t *pos) {
    size_t lo = 0, hi = q->n_series;
    while (lo < hi) {
        size_t mid = (lo + hi) / 2;
        if (q->sids[mid] < sid) lo = mid + 1;
        else hi = mid;
    }
    if (lo < q->n_series && q->sids[lo] == sid) {
        if (pos) *pos = lo;
        return 1;
    }
    return 0;
}

static int select_blocks(scan *s) {
    const ob_query *q = s->q;
    size_t cap = 256;
    s->cur = (cursor *)calloc(cap, sizeof(cursor));
    s->n_cur = 0;
    if (q->n_series == 0) return 0;
    for (int pi = 0; pi < q->n_parts; pi++) {
        ob_part *p = q->parts[pi];
        for (size_t b = 0; b < p->n_pbm; b++) {
            const obi_primary *pb = &p->pbm[b];
            /* part_iter.go:149 primary-block time prune */
            if (pb->max_ts < q->tmin || pb->min_ts > q->tmax) continue;
            /* sid prune: this primary block holds sids in [pb->sid, next.sid] */
            uint64_t hi_sid = b + 1 < p->n_pbm ? p->pbm[b + 1].sid : UINT64_MAX;
            if (q->sids[q->n_series - 1] < pb->sid || q->sids[0] > hi_sid) continue;
            obi_blockmeta *bms;
            size_t nb;
            if (obi_part_read_primary_block(p, b, &bms, &nb) != 0) return -1;
            for (size_t k = 0; k < nb; k++) {
                /* part_iter.go:218-241 findBlock */
                if (!sid_selected(q, bms[k].sid, NULL) || bms[k].ts_max < q->tmin || bms[k].ts_min > q->tmax) {
                    obi_bm_free(&bms[k]);
                    continue;
                }
                if (s->n_cur == cap) {
                    cap *= 2;
                    s->cur = (cursor *)realloc(s->cur, cap * sizeof(cursor));
                    memset(s->cur + s->n_cur, 0, (cap - s->n_cur) * sizeof(cursor));
                }
                cursor *c = &s->cur[s->n_cur++];
                c->part = pi;
                c->bm = bms[k]; /* ownership moves */
            }
            free(bms);
        }
    }
    return 0;
}

/* ------------------------------------------------------------------ block load (block.go:793-870) */
/* pkg/timestamp/range.go:143-169 FindRange (ascending case; blocks are validated ascending at write) */
static int find_range(const int64_t *ts, size_t n, int64_t minv, int64_t maxv, size_t *start, size_t *end) {
    if (n == 0) return 0;
    int asc = ts[0] <= ts[n - 1];
    if (asc && (ts[0] > maxv || ts[n - 1] < minv)) return 0;
    if (!asc && (ts[0] < minv || ts[n - 1] > maxv)) return 0;
    long st = -1, en = (long)n;
    while (st < (long)n - 1) {
        st++;
        if ((asc && ts[st] >= minv) || (!asc && ts[st] <= maxv)) break;
    }
    while (en > 0) {
        en--;
        if ((asc && ts[en] <= maxv) || (!asc && ts[en] >= minv)) break;
    }
    *start = (size_t)st;
    *end = (size_t)en;
    return st <= en;
}

static int decode_numeric(const uint8_t *src, size_t srclen, int value_type, size_t count, fcol *out) {
    out->is_float = value_type == OB_VT_FLOAT64;
    out->present = 1;
    if (srclen < 1) return -1;
    int enc = src[0];
    if (enc == OB_ENC_PLAIN) {
        /* column.go:297-301 / 335-339: fallback page -> 8-byte cells (or nil) */
        ob_bytes *cells = (ob_bytes *)malloc(sizeof(ob_bytes) * (count ? count : 1));
        ob_buf arena = {0};
        if (ob_column_decode(cells, count, value_type, src, srclen, &arena) != 0) {
            free(cells);
            ob_buf_free(&arena);
            return -1;
        }
        out->null = (uint8_t *)calloc(count ? count : 1, 1);
        if (out->is_float) out->f64 = (double *)calloc(count ? count : 1, sizeof(double));
        else out->i64 = (int64_t *)calloc(count ? count : 1, sizeof(int64_t));
        for (size_t i = 0; i < count; i++) {
            if (cells[i].len < 0) { /* batch_decode.go:108-127: nil -> AppendNull */
                out->null[i] = 1;
                continue;
            }
            if (cells[i].len < 8) {
                free(cells);
                ob_buf_free(&arena);
                return -1;
            }
            if (out->is_float) {
                uint64_t u = 0;
                for (int k = 0; k < 8; k++) u = (u << 8) | cells[i].p[k];
                memcpy(&out->f64[i], &u, 8);
            } else {
                out->i64[i] = ob_conv_bytes_to_int64(cells[i].p);
            }
        }
        free(cells);
        ob_buf_free(&arena);
        return 0;
    }
    size_t hdr = out->is_float ? 11 : 9;
    if (srclen < hdr) return -1;
    int16_t exp = 0;
    if (out->is_float) exp = (int16_t)(((uint16_t)src[1] << 8) | src[2]);
    int64_t first = ob_conv_bytes_to_int64(src + hdr - 8);
    int64_t *ints = (int64_t *)malloc(sizeof(int64_t) * (count ? count : 1));
    if (ob_int64_list_decode(ints, src + hdr, srclen - hdr, enc, first, count) != 0) {
        free(ints);
        return -1;
    }
    if (out->is_float) {
        out->f64 = (double *)malloc(sizeof(double) * (count ? count : 1));
        ob_decimal_list_to_float64(out->f64, ints, count, exp);
        free(ints);
    } else {
        out->i64 = ints;
    }
    return 0;
}

/* tag columns a cursor loads: one per predicate, then one per group-key component */
static int n_tag_cols(const ob_query *q) { return q->n_preds + q->n_keys; }

static void cursor_free(cursor *c, int n_fcols, int n_preds) {
    free(c->ts);
    free(c->ver);
    if (c->fields) {
        for (int i = 0; i < n_fcols; i++) {
            free(c->fields[i].i64);
            free(c->fields[i].f64);
            free(c->fields[i].null);
        }
        free(c->fields);
    }
    if (c->tags) {
        for (int i = 0; i < n_preds; i++) {
            free(c->tags[i].cells);
            ob_buf_free(&c->tags[i].arena);
        }
        free(c->tags);
    }
    obi_bm_free(&c->bm);
    memset(c, 0, sizeof *c);
}

/* blockCursor.loadData, block.go:793-870 (+ mustReadFrom :299-330) */
static int load_cursor(scan *s, cursor *c) {
    const ob_query *q = s->q;
    ob_part *p = q->parts[c->part];
    size_t count = (size_t)c->bm.count;
    obi_file *tsf = obi_part_file(p, "timestamps.bin", 0);
    obi_file *fv = obi_part_file(p, "fv.bin", 0);
    if (!tsf || c->bm.ts_off + c->bm.ts_size > tsf->data.len || c->bm.ver_off > c->bm.ts_size) {
        ob_set_error("timestamps block out of bounds");
        return -1;
    }
    int64_t *ts = (int64_t *)malloc(sizeof(int64_t) * (count ? count : 1));
    int64_t *ver = (int64_t *)malloc(sizeof(int64_t) * (count ? count : 1));
    const uint8_t *tsrc = tsf->data.p + c->bm.ts_off;
    /* block.go:400-418 mustDecodeTimestampsWithVersions */
    int common = c->bm.ts_enc - 4;
    if (common < OB_ENC_CONST || common > OB_ENC_DELTA_OF_DELTA ||
        ob_int64_list_decode(ts, tsrc, (size_t)c->bm.ver_off, common, c->bm.ts_min, count) != 0 ||
        ob_int64_list_decode(ver, tsrc + c->bm.ver_off, (size_t)(c->bm.ts_size - c->bm.ver_off), c->bm.ver_enc, c->bm.ver_first, count) != 0) {
        free(ts);
        free(ver);
        ob_set_error("cannot decode timestamps/versions");
        return -1;
    }
    size_t st, en;
    if (!find_range(ts, count, q->tmin, q->tmax, &st, &en)) {
        free(ts);
        free(ver);
        c->blank = 1;
        return 0;
    }
    c->n = en - st + 1;
    c->ts = (int64_t *)malloc(sizeof(int64_t) * c->n);
    c->ver = (int64_t *)malloc(sizeof(int64_t) * c->n);
    memcpy(c->ts, ts + st, sizeof(int64_t) * c->n);
    memcpy(c->ver, ver + st, sizeof(int64_t) * c->n);
    free(ts);
    free(ver);

    c->fields = (fcol *)calloc((size_t)(s->n_fcols ? s->n_fcols : 1), sizeof(fcol));
    for (int f = 0; f < s->n_fcols; f++) {
        const obi_colmeta *cm = NULL;
        for (size_t k = 0; k < c->bm.n_fields; k++)
            if (strcmp(c->bm.fields[k].name, s->fcol_names[f]) == 0) cm = &c->bm.fields[k];
        if (!cm) continue; /* block.go:801-805: ValueTypeUnknown -> all nil */
        if (cm->value_type != OB_VT_INT64 && cm->value_type != OB_VT_FLOAT64) {
            ob_set_error("aggregation over a non-numeric field");
            return -1;
        }
        if (!fv || cm->offset + cm->size > fv->data.len) {
            ob_set_error("field page out of bounds");
            return -1;
        }
        fcol full;
        memset(&full, 0, sizeof full);
        if (decode_numeric(fv->data.p + cm->offset, (size_t)cm->size, cm->value_type, count, &full) != 0) {
            free(full.i64);
            free(full.f64);
            free(full.null);
            ob_set_error("cannot decode field page");
            return -1;
        }
        fcol *o = &c->fields[f];
        o->present = 1;
        o->is_float = full.is_float;
        if (full.is_float) {
            o->f64 = (double *)malloc(sizeof(double) * c->n);
            memcpy(o->f64, full.f64 + st, sizeof(double) * c->n);
        } else {
            o->i64 = (int64_t *)malloc(sizeof(int64_t) * c->n);
            memcpy(o->i64, full.i64 + st, sizeof(int64_t) * c->n);
        }
        if (full.null) {
            o->null = (uint8_t *)malloc(c->n);
            memcpy(o->null, full.null + st, c->n);
        }
        free(full.i64);
        free(full.f64);
        free(full.null);
    }
    const int n_tcols = n_tag_cols(q);
    c->tags = (tcol *)calloc((size_t)(n_tcols ? n_tcols : 1), sizeof(tcol));
    for (int t = 0; t < n_tcols; t++) {
        const char *t_family = t < q->n_preds ? q->preds[t].family : q->keys[t - q->n_preds].family;
        const char *t_tag = t < q->n_preds ? q->preds[t].tag : q->keys[t - q->n_preds].tag;
        const obi_fammeta *fm = NULL;
        for (size_t k = 0; k < c->bm.n_fams; k++)
            if (strcmp(c->bm.fams[k].name, t_family) == 0) fm = &c->bm.fams[k];
        if (!fm) continue;
        char fn[200];
        snprintf(fn, sizeof fn, "%s.tfm", t_family);
        obi_file *tfm = obi_part_file(p, fn, 0);
        snprintf(fn, sizeof fn, "%s.tf", t_family);
        obi_file *tf = obi_part_file(p, fn, 0);
        if (!tfm || !tf || fm->offset + fm->size > tfm->data.len) {
            ob_set_error("tag family metadata out of bounds");
            return -1;
        }
        obi_colmeta *cms;
        size_t ncm;
        if (!obi_cfm_unmarshal(tfm->data.p + fm->offset, tfm->data.p + fm->offset + fm->size, &cms, &ncm)) {
            ob_set_error("cannot unmarshal columnFamilyMetadata");
            return -1;
        }
        for (size_t k = 0; k < ncm; k++) {
            if (strcmp(cms[k].name, t_tag) != 0) continue;
            if (cms[k].offset + cms[k].size > tf->data.len) {
                free(cms);
                ob_set_error("tag page out of bounds");
                return -1;
            }
            ob_bytes *cells = (ob_bytes *)malloc(sizeof(ob_bytes) * (count ? count : 1));
            if (ob_column_decode(cells, count, cms[k].value_type, tf->data.p + cms[k].offset, (size_t)cms[k].size, &c->tags[t].arena) != 0) {
                free(cells);
                free(cms);
                ob_set_error("cannot decode tag page");
                return -1;
            }
            c->tags[t].present = 1;
            c->tags[t].value_type = cms[k].value_type;
            c->tags[t].cells = (ob_bytes *)malloc(sizeof(ob_bytes) * c->n);
            memcpy(c->tags[t].cells, cells + st, sizeof(ob_bytes) * c->n);
            free(cells);
            break;
        }
        free(cms);
    }
    return 0;
}

/* ------------------------------------------------------------------ predicates */
static int pred_match(const ob_pred *pr, const tcol *tc, size_t row) {
    int have = tc->present && tc->cells[row].len >= 0;
    int cmp = 0;
    if (have) {
        const ob_bytes *cell = &tc->cells[row];
        if (pr->value_type == OB_VT_INT64) {
            if (tc->value_type != OB_VT_INT64 || cell->len != 8) have = 0;
            else {
                int64_t v = ob_conv_bytes_to_int64(cell->p);
                cmp = v < pr->i64 ? -1 : (v > pr->i64 ? 1 : 0);
            }
        } else {
            size_t la = (size_t)cell->len, lb = pr->str.len < 0 ? 0 : (size_t)pr->str.len;
            size_t m = la < lb ? la : lb;
            cmp = m ? memcmp(cell->p, pr->str.p, m) : 0;
            if (cmp == 0) cmp = la < lb ? -1 : (la > lb ? 1 : 0);
        }
    }
    switch (pr->op) {
    case OB_OP_EQ: return have && cmp == 0;
    case OB_OP_NE: return !have || cmp != 0;
    case OB_OP_LT: return have && cmp < 0;
    case OB_OP_LE: return have && cmp <= 0;
    case OB_OP_GT: return have && cmp > 0;
    case OB_OP_GE: return have && cmp >= 0;
    }
    return 0;
}

/* ------------------------------------------------------------------ aggregation state (function.go) */
typedef struct {
    int func, is_float, int_map; /* int_map: accumulator is Map[int64] (aggregation.go:342-375) */
    int64_t isum, icount, ival;
    double fsum, fcount, fval;
} slot;

static void slot_init(slot *s, int func, int field_is_float) {
    memset(s, 0, sizeof *s);
    s->func = func;
    s->is_float = field_is_float;
    s->int_map = (func == OB_AGG_COUNT) || !field_is_float;
    if (func == OB_AGG_MAX) { /* aggregation.go:169-179 minOf */
        s->ival = INT64_MIN;
        s->fval = -DBL_MAX;
    } else if (func == OB_AGG_MIN) { /* :181-191 maxOf */
        s->ival = INT64_MAX;
        s->fval = DBL_MAX;
    }
}
/* aggregation.go:290-312 fold + function.go In() */
static void slot_in_i(slot *s, int64_t v) {
    switch (s->func) {
    case OB_AGG_MEAN: s->isum = wadd(s->isum, v); s->icount++; break;
    case OB_AGG_COUNT: s->icount++; break;
    case OB_AGG_SUM: s->isum = wadd(s->isum, v); break;
    case OB_AGG_MAX: if (v > s->ival) s->ival = v; break;
    case OB_AGG_MIN: if (v < s->ival) s->ival = v; break;
    }
}
static void slot_in_f(slot *s, double v) {
    switch (s->func) {
    case OB_AGG_MEAN: s->fsum += v; s->fcount += 1; break;
    case OB_AGG_COUNT: s->fcount += 1; break;
    case OB_AGG_SUM: s->fsum += v; break;
    case OB_AGG_MAX: if (v > s->fval) s->fval = v; break;
    case OB_AGG_MIN: if (v < s->fval) s->fval = v; break;
    }
}
/* function.go Val() */
static int64_t slot_val_i(const slot *s) {
    switch (s->func) {
    case OB_AGG_MEAN: {
        if (s->icount == 0) return 0;
        int64_t v = s->isum / s->icount; /* Go int division truncates toward zero, like C */
        return v < 1 ? 1 : v;
    }
    case OB_AGG_COUNT: return s->icount;
    case OB_AGG_SUM: return s->isum;
    default: return s->ival;
    }
}
static double slot_val_f(const slot *s) {
    switch (s->func) {
    case OB_AGG_MEAN: {
        if (s->fcount == 0) return 0;
        double v = s->fsum / s->fcount;
        return v < 1 ? 1 : v;
    }
    case OB_AGG_COUNT: return s->fcount;
    case OB_AGG_SUM: return s->fsum;
    default: return s->fval;
    }
}
/* Reduce.Combine (function.go:45-48,98-100,148-150,184-188,220-228) for the per-thread-partials mode */
static void slot_combine(slot *a, const slot *b) {
    switch (a->func) {
    case OB_AGG_MEAN:
        a->isum = wadd(a->isum, b->isum);
        a->icount += b->icount;
        a->fsum += b->fsum;
        a->fcount += b->fcount;
        break;
    case OB_AGG_COUNT:
        a->icount += b->icount;
        a->fcount += b->fcount;
        break;
    case OB_AGG_SUM:
        a->isum = wadd(a->isum, b->isum);
        a->fsum += b->fsum;
        break;
    case OB_AGG_MAX:
        if (b->ival > a->ival) a->ival = b->ival;
        if (b->fval > a->fval) a->fval = b->fval;
        break;
    case OB_AGG_MIN: /* "still at sentinel" == empty */
        if (a->ival == INT64_MAX || b->ival < a->ival) a->ival = b->ival;
        if (a->fval == DBL_MAX || b->fval < a->fval) a->fval = b->fval;
        break;
    }
}

typedef struct {
    int64_t rows;
    int typed; /* slot types fixed (first non-missing block decides) */
    slot *slots;
} group;

/* ------------------------------------------------------------------ per-series merge (query.go:912-1025) */
typedef struct {
    int32_t gid;    /* group of the row's series */
    uint64_t hash;  /* comp_hash(gid, key) */
    ob_bytes key;   /* encoded key (owned) */
} comp;

typedef struct {
    scan *s;
    group *groups;   /* [n_groups]; with a group key: [n_comp], one per (series group, encoded key) in first-seen order */
    int *agg_float;  /* [n_aggs] -1 unknown, 0 int, 1 float */
    uint64_t rows_matched;
    ob_rows *rows_out; /* optional raw dump */
    size_t rows_cap;
    /* per-row group key: pkg/query/vectorized/measure/aggregation.go:193-254 -- the group of a row is found by its encoded key
     * (encode_key); new groups are appended to the insertion list and emitted in that order */
    int keyed;
    comp *comps;
    size_t n_comp, cap_comp, last_comp;
    int32_t *slots; /* open addressing over comps by hash, -1 = empty; at most half full */
    size_t slot_mask;
    ob_buf kbuf;    /* the current row's encoded key */
    int key_bad_type;
} folder;

static uint64_t comp_hash(int32_t gid, const uint8_t *p, size_t n) {
    uint64_t h = (0xcbf29ce484222325ull ^ (uint32_t)gid) * 0x100000001b3ull;
    for (size_t i = 0; i < n; i++) h = (h ^ p[i]) * 0x100000001b3ull;
    return h ^ (h >> 29);
}

/* computeKey (aggregation.go:328-337) with appendKeyComponent (groupby.go:217-254), one component per key in GroupBy order:
 * int64 -> 8 little-endian bytes (a nil cell or a block without the column: 0); string / binary -> 4-byte little-endian length,
 * then the bytes (nil: "").  -1 when a block stores a key column with another type than the key declares. */
static int encode_key(const ob_query *q, const cursor *c, size_t row, ob_buf *dst) {
    ob_buf_reset(dst);
    for (int k = 0; k < q->n_keys; k++) {
        const tcol *kc = &c->tags[q->n_preds + k];
        const ob_bytes *cell = kc->present && kc->cells[row].len >= 0 ? &kc->cells[row] : NULL;
        uint8_t b[8];
        if (q->keys[k].value_type == OB_VT_INT64) {
            if (kc->present && kc->value_type != OB_VT_INT64) return -1;
            if (cell && cell->len != 8) return -1;
            uint64_t v = cell ? (uint64_t)ob_conv_bytes_to_int64(cell->p) : 0;
            for (int i = 0; i < 8; i++) b[i] = (uint8_t)(v >> (8 * i));
            ob_buf_append(dst, b, 8);
        } else {
            if (kc->present && kc->value_type != OB_VT_STR && kc->value_type != OB_VT_BINARY) return -1;
            uint32_t n = cell ? (uint32_t)cell->len : 0;
            for (int i = 0; i < 4; i++) b[i] = (uint8_t)(n >> (8 * i));
            ob_buf_append(dst, b, 4);
            if (n) ob_buf_append(dst, cell->p, n);
        }
    }
    return 0;
}

static void slots_resize(folder *fo, size_t n_slots) {
    free(fo->slots);
    fo->slots = (int32_t *)malloc(sizeof(int32_t) * n_slots);
    for (size_t i = 0; i < n_slots; i++) fo->slots[i] = -1;
    fo->slot_mask = n_slots - 1;
    for (size_t ci = 0; ci < fo->n_comp; ci++) {
        size_t s = fo->comps[ci].hash & fo->slot_mask;
        while (fo->slots[s] >= 0) s = (s + 1) & fo->slot_mask;
        fo->slots[s] = (int32_t)ci;
    }
}

static int32_t keyed_group(folder *fo, const cursor *c, size_t row, int32_t gid) {
    const ob_query *q = fo->s->q;
    if (encode_key(q, c, row, &fo->kbuf) != 0) {
        fo->key_bad_type = 1;
        return -1;
    }
    const uint8_t *kp = fo->kbuf.p;
    const size_t kl = fo->kbuf.len; /* >= 4: every key has a component */
    if (fo->n_comp) { /* runs of equal keys are the common case */
        const comp *lc = &fo->comps[fo->last_comp];
        if (lc->gid == gid && (size_t)lc->key.len == kl && memcmp(lc->key.p, kp, kl) == 0) return (int32_t)fo->last_comp;
    }
    if (2 * (fo->n_comp + 1) > fo->slot_mask + 1) slots_resize(fo, fo->slots ? 2 * (fo->slot_mask + 1) : 1024);
    const uint64_t h = comp_hash(gid, kp, kl);
    size_t s = h & fo->slot_mask;
    for (; fo->slots[s] >= 0; s = (s + 1) & fo->slot_mask) {
        const comp *cc = &fo->comps[fo->slots[s]];
        if (cc->hash == h && cc->gid == gid && (size_t)cc->key.len == kl && memcmp(cc->key.p, kp, kl) == 0) {
            fo->last_comp = (size_t)fo->slots[s];
            return fo->slots[s];
        }
    }
    const size_t ci = fo->n_comp;
    if (ci == fo->cap_comp) {
        fo->cap_comp = fo->cap_comp ? fo->cap_comp * 2 : 16;
        fo->comps = (comp *)realloc(fo->comps, sizeof(comp) * fo->cap_comp);
        fo->groups = (group *)realloc(fo->groups, sizeof(group) * fo->cap_comp);
    }
    uint8_t *cp = (uint8_t *)malloc(kl);
    memcpy(cp, kp, kl);
    fo->comps[ci].gid = gid;
    fo->comps[ci].hash = h;
    fo->comps[ci].key.p = cp;
    fo->comps[ci].key.len = (int64_t)kl;
    memset(&fo->groups[ci], 0, sizeof(group));
    fo->groups[ci].slots = (slot *)calloc((size_t)(q->n_aggs ? q->n_aggs : 1), sizeof(slot));
    fo->slots[s] = (int32_t)ci;
    fo->n_comp++;
    fo->last_comp = ci;
    return (int32_t)ci;
}

static void fold_row(folder *fo, const cursor *c, size_t row, int32_t gid) {
    const ob_query *q = fo->s->q;
    for (int t = 0; t < q->n_preds; t++)
        if (!pred_match(&q->preds[t], &c->tags[t], row)) return;
    fo->rows_matched++;
    if (fo->rows_out) {
        ob_rows *r = fo->rows_out;
        if (r->n == fo->rows_cap) {
            fo->rows_cap = fo->rows_cap ? fo->rows_cap * 2 : 1024;
            r->sid = (uint64_t *)realloc(r->sid, sizeof(uint64_t) * fo->rows_cap);
            r->ts = (int64_t *)realloc(r->ts, sizeof(int64_t) * fo->rows_cap);
            r->version = (int64_t *)realloc(r->version, sizeof(int64_t) * fo->rows_cap);
            for (int f = 0; f < r->n_fields; f++) {
                r->i64[f] = (int64_t *)realloc(r->i64[f], sizeof(int64_t) * fo->rows_cap);
                r->f64[f] = (double *)realloc(r->f64[f], sizeof(double) * fo->rows_cap);
                r->null[f] = (uint8_t *)realloc(r->null[f], fo->rows_cap);
            }
        }
        r->sid[r->n] = c->bm.sid;
        r->ts[r->n] = c->ts[row];
        r->version[r->n] = c->ver[row];
        for (int f = 0; f < r->n_fields; f++) {
            const fcol *fc = &c->fields[f];
            int isnull = !fc->present || (fc->null && fc->null[row]);
            r->null[f][r->n] = (uint8_t)isnull;
            r->i64[f][r->n] = (!isnull && !fc->is_float) ? fc->i64[row] : 0;
            r->f64[f][r->n] = (!isnull && fc->is_float) ? fc->f64[row] : 0;
            if (fc->present) r->is_float[f] = (uint8_t)fc->is_float;
        }
        r->n++;
        return;
    }
    if (fo->keyed) {
        gid = keyed_group(fo, c, row, gid);
        if (gid < 0) return;
    }
    group *g = &fo->groups[gid];
    g->rows++;
    for (int a = 0; a < q->n_aggs; a++) {
        const fcol *fc = &c->fields[fo->s->agg_fcol[a]];
        if (!fc->present) continue; /* unknown column: all null */
        if (fo->agg_float[a] < 0) fo->agg_float[a] = fc->is_float;
        slot *sl = &g->slots[a];
        if (!(g->typed & (1 << a))) {
            slot_init(sl, q->aggs[a].func, fc->is_float);
            g->typed |= 1 << a;
        }
        if (fc->null && fc->null[row]) continue; /* aggregation.go:292-294 */
        /* a float input only reaches an int map for COUNT, which ignores the value (aggregation.go:296-304) */
        if (sl->int_map) slot_in_i(sl, fc->is_float ? 0 : fc->i64[row]);
        else slot_in_f(sl, fc->is_float ? fc->f64[row] : (double)fc->i64[row]);
    }
}

/* One series: k-way merge of its cursors ordered (ts asc, version desc); a duplicate timestamp keeps
 * the first (= highest version) row: query.go:912-942 Less, :995-1004 / query_batch.go:151-161. */
static void merge_series(folder *fo, cursor **cs, size_t k, int32_t gid) {
    if (k == 1) {
        cursor *c = cs[0];
        int have_last = 0;
        int64_t last_ts = 0;
        for (size_t i = 0; i < c->n; i++) {
            if (have_last && c->ts[i] == last_ts) continue; /* cannot happen inside one block; kept for symmetry */
            fold_row(fo, c, i, gid);
            last_ts = c->ts[i];
            have_last = 1;
        }
        return;
    }
    int have_last = 0;
    int64_t last_ts = 0;
    for (;;) {
        cursor *best = NULL;
        for (size_t i = 0; i < k; i++) {
            cursor *c = cs[i];
            if (c->idx >= c->n) continue;
            if (!best) {
                best = c;
                continue;
            }
            int64_t a = c->ts[c->idx], b = best->ts[best->idx];
            /* equal (timestamp, version) in several parts: the reference's heap leaves the winner to container/heap's
             * internal order (Less is false both ways, query.go:912-942; the first one popped is kept, :995-1004), i.e. it
             * is unspecified -- real writes never produce it with different values.  Oracle and device both define it:
             * the row of the earlier part of the query wins. */
            if (a < b || (a == b && (c->ver[c->idx] > best->ver[best->idx] ||
                                     (c->ver[c->idx] == best->ver[best->idx] && c->part < best->part))))
                best = c;
        }
        if (!best) break;
        int64_t t = best->ts[best->idx];
        if (!(have_last && t == last_ts)) {
            fold_row(fo, best, best->idx, gid);
            last_ts = t;
            have_last = 1;
        }
        best->idx++;
    }
}

static int cursor_cmp(const void *pa, const void *pb) {
    const cursor *a = *(cursor *const *)pa, *b = *(cursor *const *)pb;
    if (a->bm.sid != b->bm.sid) return a->bm.sid < b->bm.sid ? -1 : 1;
    if (a->bm.ts_min != b->bm.ts_min) return a->bm.ts_min < b->bm.ts_min ? -1 : 1;
    return a->part - b->part;
}

/* ------------------------------------------------------------------ threads */
typedef struct {
    scan *s;
    size_t next, total;
    pthread_mutex_t mu;
    int err;
    char errmsg[256];
} load_pool;

static void *load_worker(void *arg) {
    load_pool *lp = (load_pool *)arg;
    for (;;) {
        pthread_mutex_lock(&lp->mu);
        size_t i = lp->next++;
        pthread_mutex_unlock(&lp->mu);
        if (i >= lp->total) break;
        if (load_cursor(lp->s, &lp->s->cur[i]) != 0) {
            pthread_mutex_lock(&lp->mu);
            if (!lp->err) {
                lp->err = 1;
                snprintf(lp->errmsg, sizeof lp->errmsg, "%s", ob_last_error());
            }
            pthread_mutex_unlock(&lp->mu);
        }
    }
    return NULL;
}

static int load_all(scan *s, int threads) {
    load_pool lp;
    memset(&lp, 0, sizeof lp);
    lp.s = s;
    lp.total = s->n_cur;
    pthread_mutex_init(&lp.mu, NULL);
    if (threads <= 1) {
        load_worker(&lp);
    } else {
        pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)threads);
        for (int i = 0; i < threads; i++) pthread_create(&th[i], NULL, load_worker, &lp);
        for (int i = 0; i < threads; i++) pthread_join(th[i], NULL);
        free(th);
    }
    pthread_mutex_destroy(&lp.mu);
    if (lp.err) {
        ob_set_error(lp.errmsg);
        return -1;
    }
    return 0;
}

static void scan_setup(scan *s, const ob_query *q) {
    memset(s, 0, sizeof *s);
    s->q = q;
    s->fcol_names = (const char **)calloc((size_t)(q->n_aggs ? q->n_aggs : 1), sizeof(char *));
    s->agg_fcol = (int *)calloc((size_t)(q->n_aggs ? q->n_aggs : 1), sizeof(int));
    for (int a = 0; a < q->n_aggs; a++) {
        int f;
        for (f = 0; f < s->n_fcols; f++)
            if (strcmp(s->fcol_names[f], q->aggs[a].field) == 0) break;
        if (f == s->n_fcols) s->fcol_names[s->n_fcols++] = q->aggs[a].field;
        s->agg_fcol[a] = f;
    }
}
static void scan_teardown(scan *s) {
    for (size_t i = 0; i < s->n_cur; i++) cursor_free(&s->cur[i], s->n_fcols, n_tag_cols(s->q));
    free(s->cur);
    free(s->fcol_names);
    free(s->agg_fcol);
}

typedef struct {
    folder fo;
    cursor **sorted;
    size_t lo, hi; /* cursor range (whole series only) */
    scan *s;
    int do_load;
} part_job;

static void fold_range(folder *fo, cursor **sorted, size_t lo, size_t hi) {
    const ob_query *q = fo->s->q;
    size_t i = lo;
    while (i < hi) {
        size_t j = i;
        while (j < hi && sorted[j]->bm.sid == sorted[i]->bm.sid) j++;
        size_t pos = 0;
        sid_selected(q, sorted[i]->bm.sid, &pos);
        int32_t gid = q->groups ? q->groups[pos] : 0;
        merge_series(fo, sorted + i, j - i, gid);
        i = j;
    }
}

static void *part_worker(void *arg) {
    part_job *j = (part_job *)arg;
    if (j->do_load)
        for (size_t i = j->lo; i < j->hi; i++)
            if (load_cursor(j->s, j->sorted[i]) != 0) return (void *)1;
    /* drop blank cursors in place */
    size_t w = j->lo;
    for (size_t i = j->lo; i < j->hi; i++)
        if (!j->sorted[i]->blank) j->sorted[w++] = j->sorted[i];
    fold_range(&j->fo, j->sorted, j->lo, w);
    return NULL;
}

static folder folder_new(scan *s, int32_t n_groups) {
    folder fo;
    memset(&fo, 0, sizeof fo);
    fo.s = s;
    fo.groups = (group *)calloc((size_t)n_groups, sizeof(group));
    for (int32_t g = 0; g < n_groups; g++) fo.groups[g].slots = (slot *)calloc((size_t)(s->q->n_aggs ? s->q->n_aggs : 1), sizeof(slot));
    fo.agg_float = (int *)malloc(sizeof(int) * (size_t)(s->q->n_aggs ? s->q->n_aggs : 1));
    for (int a = 0; a < s->q->n_aggs; a++) fo.agg_float[a] = -1;
    return fo;
}
static void folder_free(folder *fo, int32_t n_groups) {
    if (fo->keyed) n_groups = (int32_t)fo->n_comp;
    for (int32_t g = 0; g < n_groups; g++) free(fo->groups[g].slots);
    free(fo->groups);
    free(fo->agg_float);
    for (size_t k = 0; k < fo->n_comp; k++) free((void *)fo->comps[k].key.p);
    free(fo->comps);
    free(fo->slots);
    ob_buf_free(&fo->kbuf);
}

typedef struct {
    int32_t g;
    int is_float;
    int64_t i;
    double f;
    int null;
} topent;
/* top.go:145-214: nulls lowest; ties -> earlier row (lower group index) wins */
static int top_desc;
static int top_cmp(const void *pa, const void *pb) {
    const topent *a = (const topent *)pa, *b = (const topent *)pb;
    int c; /* cmpTopVal, top.go:88-117: nulls sort LOWEST as values (last for desc, first for asc) */
    if (a->null || b->null) c = (a->null && b->null) ? 0 : (a->null ? -1 : 1);
    else if (a->is_float) c = a->f < b->f ? -1 : (a->f > b->f ? 1 : 0);
    else c = a->i < b->i ? -1 : (a->i > b->i ? 1 : 0);
    if (top_desc) c = -c;
    if (c) return c;
    return a->g < b->g ? -1 : (a->g > b->g ? 1 : 0); /* earlier row wins, top.go:62-76 */
}

int ob_query_run(const ob_query *q, ob_result *out) {
    memset(out, 0, sizeof *out);
    if (q->n_aggs > 30) {
        ob_set_error("too many aggregations");
        return -1;
    }
    if (q->n_keys < 0 || q->n_keys > OB_MAX_GROUP_KEYS) {
        ob_set_error("a group key has 1 to 4 components");
        return -1;
    }
    for (int k = 0; k < q->n_keys; k++) {
        const int vt = q->keys[k].value_type;
        if (vt != OB_VT_STR && vt != OB_VT_BINARY && vt != OB_VT_INT64) {
            ob_set_error("group key type must be string, binary or int64");
            return -1;
        }
    }
    int32_t ng = q->groups ? q->n_groups : 1;
    if (ng < 1) ng = 1;
    scan s;
    scan_setup(&s, q);
    if (select_blocks(&s) != 0) {
        scan_teardown(&s);
        return -1;
    }
    out->blocks_scanned = s.n_cur;
    for (size_t i = 0; i < s.n_cur; i++) out->rows_scanned += s.cur[i].bm.count;
    cursor **sorted = (cursor **)malloc(sizeof(cursor *) * (s.n_cur ? s.n_cur : 1));
    for (size_t i = 0; i < s.n_cur; i++) sorted[i] = &s.cur[i];
    qsort(sorted, s.n_cur, sizeof(cursor *), cursor_cmp);

    const int keyed = q->n_keys > 0;
    folder total = folder_new(&s, keyed ? 0 : ng);
    total.keyed = keyed;
    int rc = 0;
    if (q->per_thread_partials && q->threads > 1 && !keyed) { /* insertion order needs the serial fold */
        /* best-effort all-core: whole series per worker, per-thread partials, Reduce-combine in worker order */
        int nt = q->threads;
        part_job *jobs = (part_job *)calloc((size_t)nt, sizeof(part_job));
        pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)nt);
        size_t pos = 0;
        for (int t = 0; t < nt; t++) {
            size_t target = s.n_cur * (size_t)(t + 1) / (size_t)nt;
            size_t hi = target < pos ? pos : target;
            while (hi < s.n_cur && hi > 0 && hi > pos && sorted[hi]->bm.sid == sorted[hi - 1]->bm.sid) hi++;
            if (t == nt - 1) hi = s.n_cur;
            jobs[t].fo = folder_new(&s, ng);
            jobs[t].sorted = sorted;
            jobs[t].lo = pos;
            jobs[t].hi = hi;
            jobs[t].s = &s;
            jobs[t].do_load = 1;
            pos = hi;
        }
        for (int t = 0; t < nt; t++) pthread_create(&th[t], NULL, part_worker, &jobs[t]);
        for (int t = 0; t < nt; t++) {
            void *r;
            pthread_join(th[t], &r);
            if (r) rc = -1;
        }
        for (int t = 0; t < nt && rc == 0; t++) {
            total.rows_matched += jobs[t].fo.rows_matched;
            for (int32_t g = 0; g < ng; g++) {
                group *dst = &total.groups[g], *src = &jobs[t].fo.groups[g];
                dst->rows += src->rows;
                for (int a = 0; a < q->n_aggs; a++) {
                    if (!(src->typed & (1 << a))) continue;
                    if (!(dst->typed & (1 << a))) {
                        dst->slots[a] = src->slots[a];
                        dst->typed |= 1 << a;
                    } else {
                        slot_combine(&dst->slots[a], &src->slots[a]);
                    }
                }
            }
            for (int a = 0; a < q->n_aggs; a++)
                if (total.agg_float[a] < 0) total.agg_float[a] = jobs[t].fo.agg_float[a];
        }
        for (int t = 0; t < nt; t++) folder_free(&jobs[t].fo, ng);
        free(jobs);
        free(th);
    } else {
        /* reference-shaped: decode on a pool (goroutine per block), then single-threaded merge + fold */
        rc = load_all(&s, q->threads);
        if (rc == 0) {
            size_t w = 0;
            for (size_t i = 0; i < s.n_cur; i++)
                if (!sorted[i]->blank) sorted[w++] = sorted[i];
            fold_range(&total, sorted, 0, w);
        }
    }
    if (rc == 0 && total.key_bad_type) {
        ob_set_error("group key tag stored with another value type than the key declares");
        rc = -1;
    }
    if (rc != 0) {
        free(sorted);
        folder_free(&total, ng);
        scan_teardown(&s);
        return -1;
    }
    if (keyed) ng = (int32_t)total.n_comp; /* composite groups, insertion order */
    out->rows_matched = total.rows_matched;
    out->n_aggs = q->n_aggs;
    out->is_float = (uint8_t *)calloc((size_t)(q->n_aggs ? q->n_aggs : 1), 1);
    for (int a = 0; a < q->n_aggs; a++)
        out->is_float[a] = (uint8_t)(q->aggs[a].func == OB_AGG_COUNT ? 0 : (total.agg_float[a] == 1)); /* aggregation.go:425-430 */
    int32_t nrows = 0;
    for (int32_t g = 0; g < ng; g++)
        if (total.groups[g].rows > 0) nrows++;
    topent *ents = (topent *)calloc((size_t)(nrows ? nrows : 1), sizeof(topent));
    int32_t k = 0;
    for (int32_t g = 0; g < ng; g++) {
        if (total.groups[g].rows == 0) continue;
        ents[k].g = g;
        if (q->top_n > 0) {
            const slot *sl = &total.groups[g].slots[q->top_agg];
            int typed = total.groups[g].typed & (1 << q->top_agg);
            ents[k].is_float = out->is_float[q->top_agg];
            ents[k].null = !typed;
            if (typed) {
                if (sl->int_map) ents[k].i = slot_val_i(sl);
                else ents[k].f = slot_val_f(sl);
            }
        }
        k++;
    }
    if (q->top_n > 0) {
        top_desc = q->top_desc;
        qsort(ents, (size_t)nrows, sizeof(topent), top_cmp);
        if (nrows > q->top_n) nrows = q->top_n;
    }
    out->n_rows = nrows;
    if (keyed) {
        out->n_keys = q->n_keys;
        out->key = (ob_bytes *)calloc((size_t)(nrows ? nrows : 1) * (size_t)q->n_keys, sizeof(ob_bytes));
    }
    out->group_id = (int32_t *)calloc((size_t)(nrows ? nrows : 1), sizeof(int32_t));
    out->rows = (int64_t *)calloc((size_t)(nrows ? nrows : 1), sizeof(int64_t));
    size_t nv = (size_t)(nrows ? nrows : 1) * (size_t)(q->n_aggs ? q->n_aggs : 1);
    out->val_i64 = (int64_t *)calloc(nv, sizeof(int64_t));
    out->val_f64 = (double *)calloc(nv, sizeof(double));
    for (int32_t r = 0; r < nrows; r++) {
        int32_t g = ents[r].g;
        out->group_id[r] = keyed ? total.comps[g].gid : g;
        if (keyed) { /* the encoded key back into its components */
            const uint8_t *kp = total.comps[g].key.p;
            for (int k = 0; k < q->n_keys; k++) {
                size_t n = 8;
                if (q->keys[k].value_type != OB_VT_INT64) {
                    n = (size_t)kp[0] | (size_t)kp[1] << 8 | (size_t)kp[2] << 16 | (size_t)kp[3] << 24;
                    kp += 4;
                }
                uint8_t *cp = (uint8_t *)malloc(n ? n : 1);
                if (n) memcpy(cp, kp, n);
                kp += n;
                out->key[(size_t)r * (size_t)q->n_keys + (size_t)k].p = cp;
                out->key[(size_t)r * (size_t)q->n_keys + (size_t)k].len = (int64_t)n;
            }
        }
        out->rows[r] = total.groups[g].rows;
        for (int a = 0; a < q->n_aggs; a++) {
            const slot *sl = &total.groups[g].slots[a];
            size_t o = (size_t)r * (size_t)q->n_aggs + (size_t)a;
            if (!(total.groups[g].typed & (1 << a))) continue; /* never saw the column: zero value */
            if (sl->int_map) out->val_i64[o] = slot_val_i(sl);
            else out->val_f64[o] = slot_val_f(sl);
        }
    }
    free(ents);
    free(sorted);
    folder_free(&total, ng);
    scan_teardown(&s);
    return 0;
}

void ob_result_free(ob_result *r) {
    if (r->key)
        for (size_t k = 0; k < (size_t)r->n_rows * (size_t)r->n_keys; k++) free((void *)r->key[k].p);
    free(r->key);
    free(r->group_id);
    free(r->rows);
    free(r->is_float);
    free(r->val_i64);
    free(r->val_f64);
    memset(r, 0, sizeof *r);
}

int ob_scan_rows(const ob_query *q, ob_rows *out) {
    memset(out, 0, sizeof *out);
    scan s;
    scan_setup(&s, q);
    if (select_blocks(&s) != 0 || load_all(&s, q->threads) != 0) {
        scan_teardown(&s);
        return -1;
    }
    cursor **sorted = (cursor **)malloc(sizeof(cursor *) * (s.n_cur ? s.n_cur : 1));
    size_t w = 0;
    for (size_t i = 0; i < s.n_cur; i++)
        if (!s.cur[i].blank) sorted[w++] = &s.cur[i];
    qsort(sorted, w, sizeof(cursor *), cursor_cmp);
    folder fo;
    memset(&fo, 0, sizeof fo);
    fo.s = &s;
    fo.rows_out = out;
    out->n_fields = s.n_fcols;
    out->is_float = (uint8_t *)calloc((size_t)(s.n_fcols ? s.n_fcols : 1), 1);
    out->i64 = (int64_t **)calloc((size_t)(s.n_fcols ? s.n_fcols : 1), sizeof(int64_t *));
    out->f64 = (double **)calloc((size_t)(s.n_fcols ? s.n_fcols : 1), sizeof(double *));
    out->null = (uint8_t **)calloc((size_t)(s.n_fcols ? s.n_fcols : 1), sizeof(uint8_t *));
    fold_range(&fo, sorted, 0, w);
    free(sorted);
    scan_teardown(&s);
    return 0;
}

void ob_rows_free(ob_rows *r) {
    free(r->sid);
    free(r->ts);
    free(r->version);
    for (int f = 0; f < r->n_fields; f++) {
        free(r->i64[f]);
        free(r->f64[f]);
        free(r->null[f]);
    }
    free(r->i64);
    free(r->f64);
    free(r->null);
    free(r->is_float);
    memset(r, 0, sizeof *r);
}
