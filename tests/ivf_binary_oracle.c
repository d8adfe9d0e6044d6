/* ivf_binary_oracle.c -- CPU oracle of binary IVF_FLAT search by Hamming distance (the lgpu_ivf_binary_* semantics).
 *
 * Per query: the Hamming distance popcount(q XOR c) to every packed centroid; the np nearest partitions by (distance,
 * partition id), every partition when np >= nlist; every row of those partitions scored exactly, _distance =
 * popcount(q XOR x) as f32; orc_params' row-id allow bitmap and distance range [lower, upper) drop rows before the
 * top-k; results ascending by (_distance, _rowid), unused slots UINT64_MAX / +inf.  maximum_nprobes: under a prefilter,
 * a query that kept fewer than k rows is searched again over its max_nprobes nearest partitions.  refine_factor changes
 * nothing (the distances are exact).  Worker threads split the queries.  The NumPy mirror is tests/ivf_binary_oracle.py. */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../oracle/oracle.h"

/* the arithmetic of orc_hamming_u8 (hamming_oracle.c) */
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

static int keep_row(const orc_params *p, uint64_t id, uint32_t d)
{
    if (p->allow && (id >= p->allow_bits || !((p->allow[id >> 5] >> (id & 31)) & 1u))) return 0;
    if (p->has_lower && !((float)d >= p->lower)) return 0;
    if (p->has_upper && !((float)d < p->upper)) return 0;
    return 1;
}

typedef struct {
    const uint8_t *cent, *x, *q;
    const uint64_t *part_offsets, *row_ids;
    uint32_t nlist, nbytes, q0, q1;
    const orc_params *p;
    uint64_t *out_ids; float *out_dist; uint32_t *out_count;
    int err;
} job;

static void *worker(void *arg)
{
    job *j = (job *)arg;
    const orc_params *p = j->p;
    const uint32_t nlist = j->nlist, nb = j->nbytes;
    const uint32_t nprobes = p->nprobes < nlist ? p->nprobes : nlist;
    uint32_t nprobes_max = nprobes;
    if (p->allow && p->max_nprobes > nprobes) nprobes_max = p->max_nprobes < nlist ? p->max_nprobes : nlist;
    const uint64_t nrows = j->part_offsets[nlist];
    cand *parts = (cand *)malloc(sizeof(cand) * nlist);
    cand *c = (cand *)malloc(sizeof(cand) * (nrows ? nrows : 1));
    if (!parts || !c) { j->err = 1; goto done; }
    for (uint32_t qi = j->q0; qi < j->q1; qi++) {
        const uint8_t *q = j->q + (size_t)qi * nb;
        for (uint32_t l = 0; l < nlist; l++) { parts[l].d = hamming_row(q, j->cent + (size_t)l * nb, nb); parts[l].id = l; }
        qsort(parts, nlist, sizeof(cand), cand_cmp);      /* (distance, partition id) */
        uint64_t nc = 0;
        for (uint32_t np_use = nprobes;;) {
            nc = 0;
            for (uint32_t s = 0; s < np_use; s++) {
                const uint64_t a = j->part_offsets[parts[s].id], b = j->part_offsets[parts[s].id + 1];
                for (uint64_t r = a; r < b; r++) {
                    const uint32_t d = hamming_row(q, j->x + r * nb, nb);
                    if (keep_row(p, j->row_ids[r], d)) { c[nc].d = d; c[nc].id = j->row_ids[r]; nc++; }
                }
            }
            if (np_use >= nprobes_max || nc >= p->k) break;
            np_use = nprobes_max;
        }
        qsort(c, nc, sizeof(cand), cand_cmp);
        const uint32_t cnt = (uint32_t)(nc < p->k ? nc : p->k);
        for (uint32_t i = 0; i < p->k; i++) {
            j->out_ids[(size_t)qi * p->k + i] = i < cnt ? c[i].id : UINT64_MAX;
            j->out_dist[(size_t)qi * p->k + i] = i < cnt ? (float)c[i].d : INFINITY;
        }
        j->out_count[qi] = cnt;
    }
done:
    free(parts);
    free(c);
    return NULL;
}

/* centroids [nlist][nbytes], part_offsets [nlist+1], vectors [nrows][nbytes] and row_ids [nrows] in partition order,
 * queries [B][nbytes]; p->k results per query (k, nprobes, max_nprobes, has_lower / has_upper, allow / allow_bits) */
int orc_ivf_binary_search(const uint8_t *centroids, uint32_t nlist, const uint64_t *part_offsets, const uint8_t *vectors,
                          const uint64_t *row_ids, uint32_t nbytes, const uint8_t *queries, uint32_t B,
                          const orc_params *p, uint64_t *out_ids, float *out_dist, uint32_t *out_count, int nthreads)
{
    if (!p || p->k == 0 || nbytes == 0 || nlist == 0 || p->nprobes == 0) return 1;
    if (nthreads < 1) nthreads = 1;
    if ((uint32_t)nthreads > B) nthreads = B ? (int)B : 1;
    job *js = (job *)calloc((size_t)nthreads, sizeof(job));
    pthread_t *th = (pthread_t *)calloc((size_t)nthreads, sizeof(pthread_t));
    if (!js || !th) { free(js); free(th); return 1; }
    for (int t = 0; t < nthreads; t++) {
        job x = { centroids, vectors, queries, part_offsets, row_ids, nlist, nbytes,
                  (uint32_t)((uint64_t)B * t / nthreads), (uint32_t)((uint64_t)B * (t + 1) / nthreads), p,
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
