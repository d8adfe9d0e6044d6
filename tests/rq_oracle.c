/* rq_oracle.c -- CPU oracle of IVF_RQ search: the lgpu_ivf_rq_open / lgpu_search semantics.
 *
 * orc_ivf_search (oracle/oracle.c) runs the search; this file supplies IVF_RQ's arithmetic.  Per query (normalised
 * first for cosine) the rotated query rq_i = orc_dot_f32(P row i, q) and, per probed partition p,
 * q'_i = rq_i - rc_{p,i} (rc_{p,i} = orc_dot_f32(P row i, c_p)), its 4-bit grid
 *     lo = min q', delta = (max q' - lo) / 15, u_i = min(15, trunc((q'_i - lo) / delta + 0.5)), S = sum u_i,
 * qq = orc_l2_f32(rq, rc_p), and for every row of p, with ip = sum_i b_i u_i and pc = popcount(b),
 *     y = delta * (float)(2 ip - S) + lo * (float)(2 pc - dim),   est = (add + qq) + scale * y,
 * each operation rounded to f32 on its own (this file is built with -ffp-contract=off); _distance = est (l2) or 0.5 est
 * (cosine).  -0 orders below +0 in min and max.  A NaN component of q' makes lo, hi and delta NaN; a slot whose delta
 * is not finite has NaN estimates (u is 0 then, as when delta is 0), which are never returned.  The NumPy mirror is
 * tests/rq_oracle.py. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#include "../oracle/oracle.h"

/* out[v][i] = orc_dot_f32(P row i, x[v]) */
void orc_rq_rotate(const float *P, const float *x, uint64_t n, uint32_t dim, float *out)
{
    for (uint64_t v = 0; v < n; v++)
        for (uint32_t i = 0; i < dim; i++) out[v * dim + i] = orc_dot_f32(P + (size_t)i * dim, x + v * dim, dim);
}

/* one probe slot: u [dim], grid[0..2] = lo, delta, qq, *S */
void orc_rq_slot(const float *rq, const float *rc, uint32_t dim, float *qp, uint8_t *u, float *grid, uint32_t *S)
{
    float lo = INFINITY, hi = -INFINITY;
    int nan = 0;
    for (uint32_t i = 0; i < dim; i++) {
        const float d = rq[i] - rc[i];
        qp[i] = d;
        if (d != d) nan = 1;
        else {                                  /* -0 orders below +0, so the extremes do not depend on the order */
            if (d < lo || (d == lo && signbit(d))) lo = d;
            if (d > hi || (d == hi && !signbit(d))) hi = d;
        }
    }
    if (nan) lo = hi = NAN;
    const float delta = (hi - lo) / 15.0f;
    const int ongrid = delta > 0.0f && isfinite(delta);
    uint32_t s = 0;
    for (uint32_t i = 0; i < dim; i++) {
        uint32_t c = 0;
        if (ongrid) {
            const float f = (qp[i] - lo) / delta + 0.5f;
            c = (uint32_t)f;
            if (c > 15) c = 15;
        }
        u[i] = (uint8_t)c;
        s += c;
    }
    grid[0] = lo; grid[1] = delta; grid[2] = orc_l2_f32(rq, rc, dim);
    *S = s;
}

/* the reported distance of one row (code [ceil(dim / 8)] bytes, LSB first) in a slot */
float orc_rq_estimate(const uint8_t *code, float add, float scale, const uint8_t *u, const float *grid, uint32_t S,
                      uint32_t dim, int metric)
{
    int64_t ip = 0, pc = 0;
    for (uint32_t i = 0; i < dim; i++) {
        const int b = (code[i >> 3] >> (i & 7)) & 1;
        ip += b * u[i];
        pc += b;
    }
    const float t1 = grid[1] * (float)(2 * ip - (int64_t)S);
    const float t2 = grid[0] * (float)(2 * pc - (int64_t)dim);
    const float y = t1 + t2;
    const float a = add + grid[2];
    const float sy = scale * y;
    float est = a + sy;
    if (metric == ORC_COSINE) est = 0.5f * est;
    return isfinite(grid[1]) ? est : NAN;
}

/* state: the query (normalised for cosine), its rotation, the slot's q' and u */
typedef struct { orc_ivf_kind base; const float *P, *rc; const uint8_t *codes; const float *add, *scale; } rq_kind;

static void rq_prepare(const orc_ivf_kind *k, const void *q, void *state)
{
    float *qn = (float *)state;
    orc_ivf_query_f32(k, q, state);
    orc_rq_rotate(((const rq_kind *)k)->P, qn, 1, k->ix->dim, qn + k->ix->dim);
}

/* a slot whose delta is not finite gives NaN estimates, which the row filter drops */
static void rq_partition(const orc_ivf_kind *k, void *state, uint32_t part, float *dists)
{
    const rq_kind *rk = (const rq_kind *)k;
    const uint32_t dim = k->ix->dim, nb = (dim + 7) / 8;
    float *rq = (float *)state + dim, *qp = rq + dim;
    uint8_t *u = (uint8_t *)(qp + dim);
    const uint64_t a = k->ix->part_offsets[part], b = k->ix->part_offsets[part + 1];
    float grid[3];
    uint32_t S;
    orc_rq_slot(rq, rk->rc + (size_t)part * dim, dim, qp, u, grid, &S);
    for (uint64_t r = a; r < b; r++)
        dists[r - a] = orc_rq_estimate(rk->codes + r * nb, rk->add[r], rk->scale[r], u, grid, S, dim, k->ix->metric);
}

/* ix: the IVF arrays (codebook and codes_t unused); P [dim][dim]; codes [nrows][ceil(dim / 8)], add / scale [nrows]
 * in partition order */
int orc_rq_search(const orc_index *ix, const float *P, const uint8_t *codes, const float *add, const float *scale,
                  const float *queries, uint32_t B, const orc_params *p, uint64_t *out_ids, float *out_dist,
                  uint32_t *out_count, int nthreads)
{
    if (!ix || !p || p->k == 0 || ix->dim == 0 || ix->nlist == 0) return 1;
    float *rc = (float *)malloc(sizeof(float) * ix->nlist * ix->dim);
    if (!rc) return 1;
    orc_rq_rotate(P, ix->centroids, ix->nlist, ix->dim, rc);
    const rq_kind k = { { ix, sizeof(float) * ix->dim, (3 * sizeof(float) + 1) * ix->dim, rq_prepare,
                          orc_ivf_coarse_f32, rq_partition }, P, rc, codes, add, scale };
    const int err = orc_ivf_search(&k.base, queries, B, p, out_ids, out_dist, out_count, nthreads);
    free(rc);
    return err;
}
