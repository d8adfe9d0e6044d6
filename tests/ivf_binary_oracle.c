/* ivf_binary_oracle.c -- CPU oracle of binary IVF_FLAT search by Hamming distance (the lgpu_ivf_binary_* semantics).
 *
 * Per query: the Hamming distance popcount(q XOR c) to every packed centroid; the np nearest partitions by (distance,
 * partition id), every partition when np >= nlist; every row of those partitions scored exactly, _distance =
 * popcount(q XOR x) as f32; orc_params' row-id allow bitmap and distance range [lower, upper) drop rows before the
 * top-k; results ascending by (_distance, _rowid), unused slots UINT64_MAX / +inf.  maximum_nprobes: under a prefilter,
 * a query that kept fewer than k rows is searched again over its max_nprobes nearest partitions.  refine_factor changes
 * nothing (the distances are exact).  orc_ivf_search (oracle/oracle.c) runs the search.  The NumPy mirror is
 * tests/ivf_binary_oracle.py. */
#include <stdint.h>
#include <string.h>

#include "../oracle/oracle.h"

/* state: the coarse distances [nlist], then the query */
typedef struct { orc_ivf_kind base; const uint8_t *cent, *x; uint32_t nbytes; } binary_kind;

static void binary_prepare(const orc_ivf_kind *k, const void *q, void *state)
{
    memcpy((float *)state + k->ix->nlist, q, ((const binary_kind *)k)->nbytes);
}

/* Hamming distances are integers of at most 2^24 bits: exact as f32, in the order and the range tests too */
static void binary_coarse(const orc_ivf_kind *k, const void *state, uint32_t nprobes, uint32_t *parts, float *dists)
{
    const binary_kind *bk = (const binary_kind *)k;
    float *all = (float *)state;
    const uint8_t *q = (const uint8_t *)(all + k->ix->nlist);
    for (uint32_t l = 0; l < k->ix->nlist; l++)
        all[l] = (float)orc_hamming_row(q, bk->cent + (size_t)l * bk->nbytes, bk->nbytes);
    orc_nearest(all, k->ix->nlist, nprobes, parts, dists);
}

static void binary_partition(const orc_ivf_kind *k, void *state, uint32_t part, float *dists)
{
    const binary_kind *bk = (const binary_kind *)k;
    const uint8_t *q = (const uint8_t *)((float *)state + k->ix->nlist);
    const uint64_t a = k->ix->part_offsets[part], b = k->ix->part_offsets[part + 1];
    for (uint64_t r = a; r < b; r++) dists[r - a] = (float)orc_hamming_row(q, bk->x + r * bk->nbytes, bk->nbytes);
}

/* centroids [nlist][nbytes], part_offsets [nlist+1], vectors [nrows][nbytes] and row_ids [nrows] in partition order,
 * queries [B][nbytes]; p->k results per query (k, nprobes, max_nprobes, has_lower / has_upper, allow / allow_bits) */
int orc_ivf_binary_search(const uint8_t *centroids, uint32_t nlist, const uint64_t *part_offsets, const uint8_t *vectors,
                          const uint64_t *row_ids, uint32_t nbytes, const uint8_t *queries, uint32_t B,
                          const orc_params *p, uint64_t *out_ids, float *out_dist, uint32_t *out_count, int nthreads)
{
    if (!p || p->k == 0 || nbytes == 0 || nlist == 0 || p->nprobes == 0) return 1;
    orc_index ix;
    memset(&ix, 0, sizeof(ix));
    ix.nlist = nlist; ix.nrows = part_offsets[nlist]; ix.part_offsets = part_offsets; ix.row_ids = row_ids;
    const binary_kind k = { { &ix, nbytes, sizeof(float) * nlist + nbytes, binary_prepare, binary_coarse,
                              binary_partition }, centroids, vectors, nbytes };
    return orc_ivf_search(&k.base, queries, B, p, out_ids, out_dist, out_count, nthreads);
}
