/* hnsw_sq_oracle.c -- CPU oracle of IVF_HNSW_SQ search: the lgpu_ivf_hnsw_sq_open / lgpu_search semantics.
 *
 * orc_ivf_search (oracle/oracle.c) runs the search; IVF_SQ's prepare (the query, normalised for cosine, then its codes)
 * and coarse step are reused, and this file supplies the per-partition graph search [lance, recalled].  In partition p,
 * with d = IVF_SQ's f32 distance of a row's codes and the rows ordered by (d, position in the partition):
 *   upper levels: from the entry row on the top level, at each level >= 1 move to the best neighbour while it is
 *     better than the current row; the row reached starts the level below;
 *   level 0: W = the ef' best rows seen so far (ef' = max(ef, kk); ef = 0 means ceil(1.5 k)), each expanded or not,
 *     W = {start}; while W holds an unexpanded row, expand the best one: every level-0 neighbour not evaluated yet is
 *     evaluated and offered to W.  (The usual two-heap loop -- pop the nearest candidate, stop when it is farther than
 *     W's farthest -- is the same loop: the candidate heap holds every row ever admitted to W; the nearest of them is
 *     either still in W, and then it is W's best unexpanded row, or it was evicted, and then every row in W is nearer,
 *     so W has no unexpanded row left.)
 *   result R: the kk best evaluated rows (the start row and every row level 0 evaluated) that pass the row filter
 *     (orc_keep: distance_range and the allow bitmap; d is never NaN).  Traversal ignores the filter.
 * The partition callback reports R's distances and NaN for every other row, so the driver's row filter drops them
 * and its top-kk over the probes is the merge of the R lists by (_distance, _rowid).  The NumPy mirror is
 * tests/hnsw_sq_oracle.py. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../oracle/oracle.h"

#define HNSW_NONE 0xFFFFFFFFu

uint8_t orc_sq_code(float v, double lo, double hi);
void orc_sq_encode(const float *x, uint64_t n, double lo, double hi, uint8_t *out);
float orc_sq_distance(const uint8_t *a, const uint8_t *b, uint32_t dim);

typedef struct {
    orc_ivf_kind base;
    const uint8_t *codes; double lo, hi;
    uint32_t m;
    const uint8_t *levels; const uint32_t *adj0, *upper_index, *upper_adj, *entry; const uint8_t *top_level;
    uint32_t efp, kk;
    const orc_params *p;
} hnsw_kind;

typedef struct { float d; uint32_t pos; } hent;

static int hless(float da, uint32_t pa, float db, uint32_t pb) { return da < db || (da == db && pa < pb); }

static int hcmp(const void *a, const void *b)
{
    const hent *x = (const hent *)a, *y = (const hent *)b;
    return hless(x->d, x->pos, y->d, y->pos) ? -1 : (hless(y->d, y->pos, x->d, x->pos) ? 1 : 0);
}

static void hnsw_prepare(const orc_ivf_kind *k, const void *q, void *state)
{
    const hnsw_kind *h = (const hnsw_kind *)k;
    orc_ivf_query_f32(k, q, state);
    orc_sq_encode((const float *)state, k->ix->dim, h->lo, h->hi, (uint8_t *)state + sizeof(float) * k->ix->dim);
}

/* state: the query, its codes, then scratch: the per-row distances (NaN = not evaluated) and W [efp + 1] with flags */
static void hnsw_partition(const orc_ivf_kind *k, void *state, uint32_t part, float *dists)
{
    const hnsw_kind *h = (const hnsw_kind *)k;
    const uint32_t dim = k->ix->dim, m2 = 2 * h->m;
    const uint8_t *qc = (const uint8_t *)state + sizeof(float) * dim;
    const uint64_t off = k->ix->part_offsets[part], n = k->ix->part_offsets[part + 1] - off;
    const uint8_t *codes = h->codes + off * dim;
    for (uint64_t r = 0; r < n; r++) dists[r] = NAN;
#define DIST(r) (isnan(dists[r]) ? (dists[r] = orc_sq_distance(codes + (uint64_t)(r) * dim, qc, dim)) : dists[r])
    /* upper levels: the evaluated distances here are not part of R, so they go to a separate cache */
    uint32_t cur = h->entry[part];
    float dcur = orc_sq_distance(codes + (uint64_t)cur * dim, qc, dim);
    for (int L = h->top_level[part]; L >= 1; L--) {
        for (;;) {
            const uint32_t *nb = h->upper_adj + ((uint64_t)h->upper_index[off + cur] + L - 1) * h->m;
            uint32_t best = cur; float bd = dcur;
            for (uint32_t j = 0; j < h->m; j++) {
                if (nb[j] == HNSW_NONE) continue;
                const float d = orc_sq_distance(codes + (uint64_t)nb[j] * dim, qc, dim);
                if (hless(d, nb[j], bd, best)) { best = nb[j]; bd = d; }
            }
            if (best == cur) break;
            cur = best; dcur = bd;
        }
    }
    /* level 0: W sorted by (d, pos), flags in `done` */
    hent *W = (hent *)malloc(sizeof(hent) * (h->efp + 1));
    uint8_t *done = (uint8_t *)malloc(h->efp + 1);
    uint32_t wn = 1;
    W[0].d = DIST(cur); W[0].pos = cur; done[0] = 0;
    for (;;) {
        uint32_t c = 0;
        while (c < wn && done[c]) c++;
        if (c == wn) break;
        done[c] = 1;
        const uint32_t *nb = h->adj0 + (off + W[c].pos) * (uint64_t)m2;
        for (uint32_t j = 0; j < m2; j++) {
            const uint32_t v = nb[j];
            if (v == HNSW_NONE || !isnan(dists[v])) continue;      /* evaluated already */
            const float d = DIST(v);
            if (wn == h->efp && !hless(d, v, W[wn - 1].d, W[wn - 1].pos)) continue;
            uint32_t i = wn < h->efp ? wn++ : wn - 1;              /* the worst is evicted when W is full */
            while (i > 0 && hless(d, v, W[i - 1].d, W[i - 1].pos)) { W[i] = W[i - 1]; done[i] = done[i - 1]; i--; }
            W[i].d = d; W[i].pos = v; done[i] = 0;
        }
    }
#undef DIST
    free(W); free(done);
    /* R: the kk best evaluated rows that pass the row filter; every other row reports NaN */
    hent *R = (hent *)malloc(sizeof(hent) * (n ? n : 1));
    uint64_t rn = 0;
    for (uint64_t r = 0; r < n; r++)
        if (!isnan(dists[r]) && orc_keep(h->p, k->ix->row_ids[off + r], dists[r])) { R[rn].d = dists[r]; R[rn++].pos = r; }
    qsort(R, rn, sizeof(hent), hcmp);
    for (uint64_t r = 0; r < n; r++) dists[r] = NAN;
    for (uint64_t i = 0; i < rn && i < h->kk; i++) dists[R[i].pos] = R[i].d;
    free(R);
}

/* ix: the IVF arrays (codebook and codes_t unused); codes [nrows][dim]; the graph arrays as in lgpu_ivf_hnsw_sq_desc;
 * ef = 0 means ceil(1.5 k).  Returns 1 on invalid arguments (ef' above 2048 included). */
int orc_hnsw_sq_search(const orc_index *ix, const uint8_t *codes, double lo, double hi, uint32_t m,
                       const uint8_t *levels, const uint32_t *adj0, const uint32_t *upper_index,
                       const uint32_t *upper_adj, const uint32_t *entry, const uint8_t *top_level, uint32_t ef,
                       const float *queries, uint32_t B, const orc_params *p, uint64_t *out_ids, float *out_dist,
                       uint32_t *out_count, int nthreads)
{
    if (!ix || !p || p->k == 0 || ix->dim == 0 || m == 0) return 1;
    const uint32_t kk = p->refine_factor ? p->k * p->refine_factor : p->k;
    uint32_t efp = ef ? ef : (3 * p->k + 1) / 2;
    if (efp < kk) efp = kk;
    if (efp > 2048) return 1;
    const hnsw_kind k = { { ix, sizeof(float) * ix->dim, (sizeof(float) + 1) * ix->dim, hnsw_prepare,
                            orc_ivf_coarse_f32, hnsw_partition },
                          codes, lo, hi, m, levels, adj0, upper_index, upper_adj, entry, top_level, efp, kk, p };
    return orc_ivf_search(&k.base, queries, B, p, out_ids, out_dist, out_count, nthreads);
}
