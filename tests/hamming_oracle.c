/* hamming_oracle.c -- CPU oracle of binary-vector flat search by Hamming distance (the lgpu_binary_* semantics).
 *
 * _distance = popcount(q XOR x) over the row's nbytes bytes, as f32; results ascending by (_distance, _rowid);
 * orc_params' distance range [lower, upper) and row-id allow bitmap drop rows before the top-k; unused slots are
 * UINT64_MAX / +inf.  Worker threads split the queries.  The NumPy mirror is tests/hamming_oracle.py. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../oracle/oracle.h"

uint32_t orc_hamming_row(const uint8_t *q, const uint8_t *x, uint32_t nbytes)
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

typedef struct {
    const uint8_t *q, *x;
    const uint64_t *row_ids;
    const orc_params *p;
    uint64_t n;
    uint32_t nbytes;
    uint32_t *out_d;            /* hamming_u8: [B][n] */
    uint64_t *out_ids;          /* flat search */
    float *out_dist;
    uint32_t *out_count;
} job;

static int hamming_range(void *arg, uint64_t b0, uint64_t b1)
{
    const job *j = (const job *)arg;
    for (uint64_t b = b0; b < b1; b++)
        for (uint64_t r = 0; r < j->n; r++)
            j->out_d[b * j->n + r] = orc_hamming_row(j->q + b * j->nbytes, j->x + r * j->nbytes, j->nbytes);
    return 0;
}

/* per query: all distances, the k-th smallest by a histogram over [0, 8 nbytes], then the top-k of the rows up to it
 * (the distances are integers of at most 2^24: exact as f32) */
static int search_range(void *arg, uint64_t b0, uint64_t b1)
{
    const job *j = (const job *)arg;
    const orc_params *p = j->p;
    const uint32_t k = p->k, maxd = 8 * j->nbytes;
    uint32_t *d = (uint32_t *)malloc((j->n ? j->n : 1) * sizeof(uint32_t));
    uint64_t *hist = (uint64_t *)malloc(((size_t)maxd + 1) * sizeof(uint64_t));
    orc_topk h = { (orc_cand *)malloc(sizeof(orc_cand) * k), 0, k };
    const int err = !d || !hist || !h.a;
    for (uint64_t b = b0; b < b1 && !err; b++) {
        const uint8_t *q = j->q + b * j->nbytes;
        memset(hist, 0, ((size_t)maxd + 1) * sizeof(uint64_t));
        for (uint64_t r = 0; r < j->n; r++) {
            d[r] = orc_hamming_row(q, j->x + r * j->nbytes, j->nbytes);
            if (orc_keep(p, j->row_ids ? j->row_ids[r] : r, (float)d[r])) hist[d[r]]++;
            else d[r] = UINT32_MAX;
        }
        uint32_t t = maxd;                                   /* smallest t with count(d <= t) >= k */
        uint64_t acc = 0;
        for (uint32_t v = 0; v <= maxd; v++) { acc += hist[v]; if (acc >= k) { t = v; break; } }
        h.n = 0;
        for (uint64_t r = 0; r < j->n; r++)
            if (d[r] <= t) orc_topk_offer(&h, (float)d[r], j->row_ids ? j->row_ids[r] : r, r);
        orc_topk_emit(p, &h, j->out_ids + b * k, j->out_dist + b * k, j->out_count + b);
    }
    free(d); free(hist); free(h.a);
    return err;
}

/* out[b][r] = popcount(queries[b] XOR vectors[r]) over nbytes bytes */
int orc_hamming_u8(const uint8_t *queries, uint32_t B, const uint8_t *vectors, uint64_t n, uint32_t nbytes,
                   uint32_t *out, int nthreads)
{
    job j;
    memset(&j, 0, sizeof(j));
    j.q = queries; j.x = vectors; j.n = n; j.nbytes = nbytes; j.out_d = out;
    return orc_parallel(B, nthreads, hamming_range, &j);
}

/* flat search by Hamming distance: p->k results per query (k, has_lower/has_upper, allow/allow_bits are used) */
int orc_flat_search_u8(const uint8_t *vectors, uint64_t n, uint32_t nbytes, const uint64_t *row_ids,
                       const uint8_t *queries, uint32_t B, const orc_params *p, uint64_t *out_ids, float *out_dist,
                       uint32_t *out_count, int nthreads)
{
    if (!p || p->k == 0 || nbytes == 0) return 1;
    job j;
    memset(&j, 0, sizeof(j));
    j.q = queries; j.x = vectors; j.row_ids = row_ids; j.p = p; j.n = n; j.nbytes = nbytes;
    j.out_ids = out_ids; j.out_dist = out_dist; j.out_count = out_count;
    return orc_parallel(B, nthreads, search_range, &j);
}
