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
 * lancedb_b200/csrc/pq4_scan.cu.  orc_ivf_search (oracle/oracle.c) runs the search around them.  The NumPy mirror is
 * tests/pq4_oracle.py. */
#include <math.h>
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

/* state: the query (normalised for cosine), then the slot's u8 table */
static void pq4_kind_partition(const orc_ivf_kind *k, void *state, uint32_t part, float *dists)
{
    const float *qn = (const float *)state;
    pq4_partition(k->ix, qn, part, (uint8_t *)(qn + k->ix->dim), dists);
}

int orc_pq4_search(const orc_index *ix, const float *queries, uint32_t B, const orc_params *p, uint64_t *out_ids,
                   float *out_dist, uint32_t *out_count, int nthreads)
{
    if (!ix || !p || p->k == 0 || ix->dim == 0 || ix->m < 2 || ix->m % 2) return 1;
    const orc_ivf_kind k = { ix, sizeof(float) * ix->dim, sizeof(float) * ix->dim + (size_t)ix->m * 16,
                             orc_ivf_query_f32, orc_ivf_coarse_f32, pq4_kind_partition };
    return orc_ivf_search(&k, queries, B, p, out_ids, out_dist, out_count, nthreads);
}
