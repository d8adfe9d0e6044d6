/* sq_oracle.c -- CPU oracle of IVF_SQ search: the lgpu_ivf_sq_open / lgpu_search semantics.
 *
 * orc_ivf_search (oracle/oracle.c) runs the search; this file supplies IVF_SQ's arithmetic.  Per query (normalised
 * first for cosine) the codes q_i = sat_u8(((double)v - lo) * 255 / (hi - lo)) (left to right in f64, truncated toward
 * zero, NaN -> 0, all 0 when lo == hi); for every row of a probed partition
 *     _distance = (float) sum_i (k_i - q_i)^2,
 * the sum exact in integers, one rounding to nearest f32 (never NaN).  The NumPy mirror is tests/sq_oracle.py. */
#include <stdint.h>

#include "../oracle/oracle.h"

uint8_t orc_sq_code(float v, double lo, double hi)
{
    if (!(hi != lo)) return 0;
    const double t = ((double)v - lo) * 255.0 / (hi - lo);
    if (!(t > 0.0)) return 0;                  /* negative, zero, NaN */
    if (t >= 255.0) return 255;
    return (uint8_t)t;                         /* truncation toward zero */
}

void orc_sq_encode(const float *x, uint64_t n, double lo, double hi, uint8_t *out)
{
    for (uint64_t i = 0; i < n; i++) out[i] = orc_sq_code(x[i], lo, hi);
}

float orc_sq_distance(const uint8_t *a, const uint8_t *b, uint32_t dim)
{
    uint64_t s = 0;
    for (uint32_t i = 0; i < dim; i++) {
        const int64_t d = (int64_t)a[i] - (int64_t)b[i];
        s += (uint64_t)(d * d);
    }
    return (float)s;
}

/* state: the query (normalised for cosine), then its codes */
typedef struct { orc_ivf_kind base; const uint8_t *codes; double lo, hi; } sq_kind;

static void sq_prepare(const orc_ivf_kind *k, const void *q, void *state)
{
    const sq_kind *sq = (const sq_kind *)k;
    orc_ivf_query_f32(k, q, state);
    orc_sq_encode((const float *)state, k->ix->dim, sq->lo, sq->hi, (uint8_t *)state + sizeof(float) * k->ix->dim);
}

static void sq_partition(const orc_ivf_kind *k, void *state, uint32_t part, float *dists)
{
    const uint32_t dim = k->ix->dim;
    const uint8_t *qc = (const uint8_t *)state + sizeof(float) * dim, *codes = ((const sq_kind *)k)->codes;
    const uint64_t a = k->ix->part_offsets[part], b = k->ix->part_offsets[part + 1];
    for (uint64_t r = a; r < b; r++) dists[r - a] = orc_sq_distance(codes + r * dim, qc, dim);
}

/* ix: the IVF arrays (codebook and codes_t unused); codes [nrows][dim] row codes in partition order */
int orc_sq_search(const orc_index *ix, const uint8_t *codes, double lo, double hi, const float *queries, uint32_t B,
                  const orc_params *p, uint64_t *out_ids, float *out_dist, uint32_t *out_count, int nthreads)
{
    if (!ix || !p || p->k == 0 || ix->dim == 0) return 1;
    const sq_kind k = { { ix, sizeof(float) * ix->dim, (sizeof(float) + 1) * ix->dim, sq_prepare, orc_ivf_coarse_f32,
                          sq_partition }, codes, lo, hi };
    return orc_ivf_search(&k.base, queries, B, p, out_ids, out_dist, out_count, nthreads);
}
