/* pq4_oracle.c -- CPU oracle of 4-bit IVF_PQ search: lgpu_index_open with nbits = 4, then lgpu_search.
 *
 * The index is an orc_index whose codebook is [m][16][dim/m] and whose codes_t holds, per partition, [m/2][n_p]
 * packed bytes at byte offset part_offsets[p] * m/2 (byte j: sub-vector 2j's code in bits 0-3, 2j+1's in bits 4-7).
 * Per query (normalised first for cosine, orc_normalize_f32): the nprobes nearest partitions by orc_find_partitions (a
 * partition whose centroid distance is NaN is not probed, as the GPU's coarse step leaves such slots unused).  Per
 * probed partition p, with r = q - c_p (l2, cosine) or q (dot):
 *   T[i][j]  = orc_l2_subvec(r_i, codeword j of sub-space i), or 1 - orc_dot_f32(...) for dot (orc_build_lut's
 *              arithmetic on the 16 codewords)
 *   qmin     = min T, qmax = max_{i < m-1} (max_j T[i][j] + max_j T[i+1][j]), both skipping NaN   [lance, recalled]
 *   Q[i][j]  = pq4_quant(T[i][j])                                                                 [lance, recalled]
 *   d        = pq4_distance(S = sum_i Q[i][code_i])                                               [lance, recalled]
 * The three recalled steps are one function each here (pq4_fold, orc_pq4_quant, orc_pq4_distance) and in
 * lancedb_b200/csrc/pq4_scan.cu.  A NaN d is never returned; distance_range [lower, upper) on d and the row-id allow
 * bitmap drop rows before the top-k; maximum_nprobes (under a prefilter) searches a query again over its max_nprobes
 * nearest partitions when it found fewer than k rows; refine_factor keeps the k * refine_factor best and re-ranks them by
 * orc_distance_f32 on the raw query and vectors.  Results ascend by (_distance, _rowid); unused slots are
 * UINT64_MAX / +inf.  Worker threads split the queries.  The NumPy mirror is tests/pq4_oracle.py. */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../oracle/oracle.h"

/* ((t - qmin) * 255) / (qmax - qmin), each op rounded to f32, rounded half away from zero, saturating `as u8` */
uint8_t orc_pq4_quant(float t, float qmin, float qmax)
{
    const float a = t - qmin;
    const float b = a * 255.0f;
    const float c = qmax - qmin;
    const float r = roundf(b / c);
    if (!(r > 0.0f)) return 0;                 /* negative, zero, NaN */
    if (r >= 255.0f) return 255;
    return (uint8_t)r;
}

/* ((float) S * (qmax - qmin)) / 255 + qmin * (float) m, then the 8-bit path's finish (cosine 0.5 d, dot d - (m - 1)) */
float orc_pq4_distance(uint32_t S, float qmin, float qmax, uint32_t m, int metric)
{
    const float range = qmax - qmin;
    const float a = (float)S * range;
    const float b = a / 255.0f;
    const float c = qmin * (float)m;
    const float d = b + c;
    if (metric == ORC_COSINE) return d * 0.5f;
    if (metric == ORC_DOT) return d - (float)(m - 1);
    return d;
}

/* qmin over every entry; qmax over the adjacent sub-space pairs of the row maxima; NaN skipped (an all-NaN fold gives
 * +inf / -inf) */
static void pq4_fold(const float *T, uint32_t m, float *qmin, float *qmax)
{
    float lo = INFINITY, hi = -INFINITY, prev = -INFINITY;
    for (uint32_t i = 0; i < m; i++) {
        float mx = -INFINITY;
        for (int j = 0; j < 16; j++) {
            const float v = T[i * 16 + j];
            if (v < lo) lo = v;
            if (v > mx) mx = v;
        }
        if (i > 0) {
            const float w = prev + mx;
            if (w > hi) hi = w;
        }
        prev = mx;
    }
    *qmin = lo; *qmax = hi;
}

/* the u8 table Q [m][16] and (qmin, qmax) of one probe slot; qn: the query, normalised for cosine */
void orc_pq4_tables(const orc_index *ix, const float *qn, uint32_t part, uint8_t *Q, float *qmm)
{
    const uint32_t m = ix->m, dsub = ix->dim / m;
    float *r = (float *)malloc(sizeof(float) * ix->dim);
    float *T = (float *)malloc(sizeof(float) * m * 16);
    if (!r || !T) { free(r); free(T); return; }
    if (ix->metric == ORC_DOT) {
        memcpy(r, qn, sizeof(float) * ix->dim);
    } else {
        const float *c = ix->centroids + (size_t)part * ix->dim;
        for (uint32_t t = 0; t < ix->dim; t++) r[t] = qn[t] - c[t];
    }
    for (uint32_t i = 0; i < m; i++)
        for (uint32_t j = 0; j < 16; j++) {
            const float *cw = ix->codebook + ((size_t)i * 16 + j) * dsub;
            T[i * 16 + j] = ix->metric == ORC_DOT ? 1.0f - orc_dot_f32(r + (size_t)i * dsub, cw, dsub)
                                                  : orc_l2_subvec(r + (size_t)i * dsub, cw, dsub);
        }
    pq4_fold(T, m, &qmm[0], &qmm[1]);
    for (uint32_t x = 0; x < m * 16; x++) Q[x] = orc_pq4_quant(T[x], qmm[0], qmm[1]);
    free(r); free(T);
}

/* d of every row of partition `part` (length n_p); qn normalised for cosine */
static void pq4_partition(const orc_index *ix, const float *qn, uint32_t part, uint8_t *Q, float *dists)
{
    const uint32_t m = ix->m, mh = m / 2;
    const uint64_t off = ix->part_offsets[part], n = ix->part_offsets[part + 1] - off;
    float qmm[2];
    orc_pq4_tables(ix, qn, part, Q, qmm);
    const uint8_t *codes = ix->codes_t + off * mh;
    for (uint64_t r = 0; r < n; r++) {
        uint32_t S = 0;
        for (uint32_t j = 0; j < mh; j++) {
            const uint8_t b = codes[(size_t)j * n + r];
            S += Q[(2 * j) * 16 + (b & 15)] + Q[(2 * j + 1) * 16 + (b >> 4)];
        }
        dists[r] = orc_pq4_distance(S, qmm[0], qmm[1], m, ix->metric);
    }
}

void orc_pq4_partition_distances(const orc_index *ix, const float *q, uint32_t part, float *dists)
{
    float *qn = (float *)malloc(sizeof(float) * ix->dim);
    uint8_t *Q = (uint8_t *)malloc((size_t)ix->m * 16);
    if (!qn || !Q) { free(qn); free(Q); return; }
    if (ix->metric == ORC_COSINE) orc_normalize_f32(q, ix->dim, qn);
    else memcpy(qn, q, sizeof(float) * ix->dim);
    pq4_partition(ix, qn, part, Q, dists);
    free(qn); free(Q);
}

typedef struct { float d; uint64_t id, pos; } cand;

static int cand_cmp(const void *a, const void *b)
{
    const cand *x = (const cand *)a, *y = (const cand *)b;
    if (x->d < y->d) return -1;
    if (x->d > y->d) return 1;
    return x->id < y->id ? -1 : (x->id > y->id ? 1 : 0);
}

static int keep_row(const orc_params *p, uint64_t id, float d)
{
    if (d != d) return 0;
    if (p->allow && (id >= p->allow_bits || !((p->allow[id >> 5] >> (id & 31)) & 1u))) return 0;
    if (p->has_lower && !(d >= p->lower)) return 0;
    if (p->has_upper && !(d < p->upper)) return 0;
    return 1;
}

typedef struct {
    const orc_index *ix;
    const float *queries;
    uint32_t q0, q1;
    const orc_params *p;
    uint64_t *out_ids; float *out_dist; uint32_t *out_count;
    int err;
} job;

static void *worker(void *arg)
{
    job *j = (job *)arg;
    const orc_index *ix = j->ix;
    const orc_params *p = j->p;
    const uint32_t dim = ix->dim, nlist = ix->nlist;
    const uint32_t nprobes = p->nprobes < nlist ? p->nprobes : nlist;
    uint32_t nprobes_max = nprobes;
    if (p->allow && p->max_nprobes > nprobes) nprobes_max = p->max_nprobes < nlist ? p->max_nprobes : nlist;
    const uint32_t kk = p->refine_factor ? p->k * p->refine_factor : p->k;
    size_t max_part = 1;
    for (uint32_t q = 0; q < nlist; q++) {
        const size_t n = ix->part_offsets[q + 1] - ix->part_offsets[q];
        if (n > max_part) max_part = n;
    }
    float *qn = (float *)malloc(sizeof(float) * (dim ? dim : 1));
    uint8_t *Q = (uint8_t *)malloc((size_t)ix->m * 16);
    float *dists = (float *)malloc(sizeof(float) * max_part);
    uint32_t *parts = (uint32_t *)malloc(sizeof(uint32_t) * (nlist ? nlist : 1));
    float *pd = (float *)malloc(sizeof(float) * (nlist ? nlist : 1));
    cand *c = (cand *)malloc(sizeof(cand) * (ix->nrows ? ix->nrows : 1));
    if (!qn || !Q || !dists || !parts || !pd || !c) { j->err = 1; goto done; }
    for (uint32_t qi = j->q0; qi < j->q1; qi++) {
        const float *q = j->queries + (size_t)qi * dim;
        if (ix->metric == ORC_COSINE) orc_normalize_f32(q, dim, qn);
        else memcpy(qn, q, sizeof(float) * dim);
        uint64_t nc = 0;
        for (uint32_t np_use = nprobes;;) {
            orc_find_partitions(ix, qn, np_use, parts, pd, NULL);
            nc = 0;
            for (uint32_t s = 0; s < np_use; s++) {
                if (pd[s] != pd[s]) continue;
                const uint64_t a = ix->part_offsets[parts[s]], b = ix->part_offsets[parts[s] + 1];
                if (a == b) continue;
                pq4_partition(ix, qn, parts[s], Q, dists);
                for (uint64_t r = a; r < b; r++) {
                    const float d = dists[r - a];
                    if (keep_row(p, ix->row_ids[r], d)) { c[nc].d = d; c[nc].id = ix->row_ids[r]; c[nc].pos = r; nc++; }
                }
            }
            if (np_use >= nprobes_max || nc >= p->k) break;
            np_use = nprobes_max;
        }
        qsort(c, nc, sizeof(cand), cand_cmp);
        if (nc > kk) nc = kk;
        if (p->refine_factor && ix->vectors) {
            for (uint64_t i = 0; i < nc; i++) c[i].d = orc_distance_f32(ix->metric, q, ix->vectors + c[i].pos * dim, dim);
            qsort(c, nc, sizeof(cand), cand_cmp);
        }
        const uint32_t cnt = (uint32_t)(nc < p->k ? nc : p->k);
        for (uint32_t i = 0; i < p->k; i++) {
            j->out_ids[(size_t)qi * p->k + i] = i < cnt ? c[i].id : UINT64_MAX;
            j->out_dist[(size_t)qi * p->k + i] = i < cnt ? c[i].d : INFINITY;
        }
        j->out_count[qi] = cnt;
    }
done:
    free(qn); free(Q); free(dists); free(parts); free(pd); free(c);
    return NULL;
}

int orc_pq4_search(const orc_index *ix, const float *queries, uint32_t B, const orc_params *p, uint64_t *out_ids,
                   float *out_dist, uint32_t *out_count, int nthreads)
{
    if (!ix || !p || p->k == 0 || ix->dim == 0 || ix->m < 2 || ix->m % 2) return 1;
    if (nthreads < 1) nthreads = 1;
    if ((uint32_t)nthreads > B) nthreads = B ? (int)B : 1;
    job *js = (job *)calloc((size_t)nthreads, sizeof(job));
    pthread_t *th = (pthread_t *)calloc((size_t)nthreads, sizeof(pthread_t));
    if (!js || !th) { free(js); free(th); return 1; }
    for (int t = 0; t < nthreads; t++) {
        job x = { ix, queries, (uint32_t)((uint64_t)B * t / nthreads), (uint32_t)((uint64_t)B * (t + 1) / nthreads), p,
                  out_ids, out_dist, out_count, 0 };
        js[t] = x;
        if (pthread_create(&th[t], NULL, worker, &js[t]) != 0) { worker(&js[t]); th[t] = 0; }
    }
    int rc = 0;
    for (int t = 0; t < nthreads; t++) {
        if (th[t]) pthread_join(th[t], NULL);
        rc |= js[t].err;
    }
    free(js);
    free(th);
    return rc;
}
