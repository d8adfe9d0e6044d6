/* hamming_oracle.c -- CPU oracle of binary-vector flat search by Hamming distance (the lgpu_binary_* semantics).
 *
 * _distance = popcount(q XOR x) over the row's nbytes bytes, as f32; results ascending by (_distance, _rowid);
 * orc_params' distance range [lower, upper) and row-id allow bitmap drop rows before the top-k; unused slots are
 * UINT64_MAX / +inf.  Worker threads split the queries.  The NumPy mirror is tests/hamming_oracle.py. */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../oracle/oracle.h"

static uint32_t hamming_row(const uint8_t *q, const uint8_t *x, uint32_t nbytes)
{
    uint32_t d = 0, i = 0;
    for (; i + 8 <= nbytes; i += 8) {
        uint64_t a, b;
        memcpy(&a, q + i, 8);
        memcpy(&b, x + i, 8);
        d += (uint32_t)__builtin_popcountll(a ^ b);
    }
    for (; i < nbytes; i++) d += (uint32_t)__builtin_popcount((unsigned)(q[i] ^ x[i]));
    return d;
}

typedef struct { uint32_t d; uint64_t id; } cand;

static int cand_cmp(const void *a, const void *b)
{
    const cand *x = (const cand *)a, *y = (const cand *)b;
    if (x->d != y->d) return x->d < y->d ? -1 : 1;
    return x->id < y->id ? -1 : (x->id > y->id ? 1 : 0);
}

typedef struct {
    const uint8_t *q, *x;
    const uint64_t *row_ids;
    const orc_params *p;
    uint64_t n;
    uint32_t B, nbytes, q0, q1;
    uint32_t *out_d;            /* hamming_u8: [B][n] */
    uint64_t *out_ids;          /* flat search */
    float *out_dist;
    uint32_t *out_count;
    int rc;
} job;

static void *hamming_worker(void *arg)
{
    job *j = (job *)arg;
    for (uint32_t b = j->q0; b < j->q1; b++)
        for (uint64_t r = 0; r < j->n; r++)
            j->out_d[(size_t)b * j->n + r] = hamming_row(j->q + (size_t)b * j->nbytes, j->x + r * j->nbytes, j->nbytes);
    return NULL;
}

static int keep_row(const orc_params *p, uint64_t id, uint32_t d)
{
    if (p->allow && (id >= p->allow_bits || !((p->allow[id >> 5] >> (id & 31)) & 1u))) return 0;
    if (p->has_lower && !((float)d >= p->lower)) return 0;
    if (p->has_upper && !((float)d < p->upper)) return 0;
    return 1;
}

/* per query: all distances, the k-th smallest by a histogram over [0, 8 nbytes], then the rows up to it sorted by
 * (distance, id) */
static void *search_worker(void *arg)
{
    job *j = (job *)arg;
    const orc_params *p = j->p;
    const uint32_t k = p->k, maxd = 8 * j->nbytes;
    uint32_t *d = (uint32_t *)malloc((j->n ? j->n : 1) * sizeof(uint32_t));
    uint64_t *hist = (uint64_t *)malloc(((size_t)maxd + 1) * sizeof(uint64_t));
    if (!d || !hist) { free(d); free(hist); j->rc = 1; return NULL; }
    for (uint32_t b = j->q0; b < j->q1; b++) {
        const uint8_t *q = j->q + (size_t)b * j->nbytes;
        memset(hist, 0, ((size_t)maxd + 1) * sizeof(uint64_t));
        for (uint64_t r = 0; r < j->n; r++) {
            const uint64_t id = j->row_ids ? j->row_ids[r] : r;
            d[r] = hamming_row(q, j->x + r * j->nbytes, j->nbytes);
            if (keep_row(p, id, d[r])) hist[d[r]]++;
            else d[r] = UINT32_MAX;
        }
        uint32_t t = maxd;                                   /* smallest t with count(d <= t) >= k */
        uint64_t acc = 0;
        for (uint32_t v = 0; v <= maxd; v++) { acc += hist[v]; if (acc >= k) { t = v; break; } }
        uint64_t m = 0;
        for (uint32_t v = 0; v <= t; v++) m += hist[v];
        cand *c = (cand *)malloc((m ? m : 1) * sizeof(cand));
        if (!c) { j->rc = 1; break; }
        uint64_t nc = 0;
        for (uint64_t r = 0; r < j->n; r++)
            if (d[r] <= t) { c[nc].d = d[r]; c[nc].id = j->row_ids ? j->row_ids[r] : r; nc++; }
        qsort(c, nc, sizeof(cand), cand_cmp);
        const uint32_t cnt = (uint32_t)(nc < k ? nc : k);
        for (uint32_t i = 0; i < k; i++) {
            j->out_ids[(size_t)b * k + i] = i < cnt ? c[i].id : UINT64_MAX;
            j->out_dist[(size_t)b * k + i] = i < cnt ? (float)c[i].d : INFINITY;
        }
        j->out_count[b] = cnt;
        free(c);
    }
    free(d);
    free(hist);
    return NULL;
}

static int run_jobs(job *proto, int nthreads, void *(*fn)(void *))
{
    if (nthreads < 1) nthreads = 1;
    if ((uint32_t)nthreads > proto->B) nthreads = proto->B ? (int)proto->B : 1;
    job *js = (job *)calloc((size_t)nthreads, sizeof(job));
    pthread_t *th = (pthread_t *)calloc((size_t)nthreads, sizeof(pthread_t));
    if (!js || !th) { free(js); free(th); return 1; }
    int rc = 0;
    for (int t = 0; t < nthreads; t++) {
        js[t] = *proto;
        js[t].q0 = (uint32_t)((uint64_t)proto->B * t / nthreads);
        js[t].q1 = (uint32_t)((uint64_t)proto->B * (t + 1) / nthreads);
        js[t].rc = 0;
        if (pthread_create(&th[t], NULL, fn, &js[t]) != 0) { fn(&js[t]); th[t] = 0; }
    }
    for (int t = 0; t < nthreads; t++) {
        if (th[t]) pthread_join(th[t], NULL);
        rc |= js[t].rc;
    }
    free(js);
    free(th);
    return rc;
}

/* out[b][r] = popcount(queries[b] XOR vectors[r]) over nbytes bytes */
int orc_hamming_u8(const uint8_t *queries, uint32_t B, const uint8_t *vectors, uint64_t n, uint32_t nbytes,
                   uint32_t *out, int nthreads)
{
    job j;
    memset(&j, 0, sizeof(j));
    j.q = queries; j.x = vectors; j.n = n; j.B = B; j.nbytes = nbytes; j.out_d = out;
    return run_jobs(&j, nthreads, hamming_worker);
}

/* flat search by Hamming distance: p->k results per query (k, has_lower/has_upper, allow/allow_bits are used) */
int orc_flat_search_u8(const uint8_t *vectors, uint64_t n, uint32_t nbytes, const uint64_t *row_ids,
                       const uint8_t *queries, uint32_t B, const orc_params *p, uint64_t *out_ids, float *out_dist,
                       uint32_t *out_count, int nthreads)
{
    if (!p || p->k == 0 || nbytes == 0) return 1;
    job j;
    memset(&j, 0, sizeof(j));
    j.q = queries; j.x = vectors; j.row_ids = row_ids; j.p = p; j.n = n; j.B = B; j.nbytes = nbytes;
    j.out_ids = out_ids; j.out_dist = out_dist; j.out_count = out_count;
    return run_jobs(&j, nthreads, search_worker);
}
