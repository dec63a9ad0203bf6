/* krag_demo.c -- the C ABI end to end from plain C (what a cgo host does, INTEGRATION.md section 2):
 * create an index, add a few nodes (dense rows + term lists), commit, run the hybrid /retrieve path, print the result.
 *
 *   gcc -std=c99 -Iinclude examples/krag_demo.c -o krag_demo -Lkaito_b200 -lkaito_rag -Wl,-rpath,$PWD/kaito_b200 -lm
 *   ./krag_demo            # needs an sm_90 (H100) GPU: krag_init fails with KRAG_E_NO_DEVICE otherwise (no CPU fallback)
 */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>

#include "kaito_rag.h"

#define CHECK(call)                                                                              \
    do {                                                                                         \
        int32_t rc_ = (call);                                                                    \
        if (rc_ != KRAG_OK) { fprintf(stderr, "%s -> %d: %s\n", #call, (int)rc_, krag_last_error()); return 1; } \
    } while (0)

enum { N = 6, DIM = 8, VOCAB = 16, K = 3 };

int main(void)
{
    krag_config cfg = {0};
    cfg.device_id = 0; cfg.world_size = 1; cfg.dense_mode = KRAG_DENSE_AUTO;
    krag_ctx* ctx = NULL;
    CHECK(krag_init(&cfg, &ctx));
    krag_index* ix = NULL;
    CHECK(krag_index_create(ctx, "demo", DIM, &ix));

    /* six unit vectors and their term lists (term id, tf); node ids are the host's (the service uses docstore ordinals) */
    float vecs[N * DIM];
    uint64_t ids[N];
    for (int i = 0; i < N; ++i) {
        double norm = 0.0;
        for (int j = 0; j < DIM; ++j) { vecs[i * DIM + j] = (float)sin(0.7 * (i + 1) * (j + 1)); norm += vecs[i * DIM + j] * vecs[i * DIM + j]; }
        for (int j = 0; j < DIM; ++j) vecs[i * DIM + j] /= (float)sqrt(norm);
        ids[i] = (uint64_t)i;
    }
    const int64_t term_off[N + 1] = {0, 2, 4, 6, 8, 10, 12};
    const uint32_t term_ids[12] = {1, 2, 2, 3, 3, 4, 1, 4, 5, 6, 1, 6};
    const uint16_t term_tf[12] = {1, 2, 1, 1, 3, 1, 1, 1, 2, 1, 1, 1};
    const uint32_t doc_len[N] = {3, 2, 4, 2, 3, 2};
    CHECK(krag_index_add(ix, N, ids, vecs, term_off, term_ids, term_tf, doc_len));
    CHECK(krag_index_commit(ix, VOCAB));          /* postings are built once here; the reference rebuilds BM25 per query */

    /* HybridRetriever._aretrieve: the query is node 2's vector, the query terms are {3, 4} */
    const uint32_t q_terms[2] = {3, 4};
    const int32_t q_off[2] = {0, 2};
    double final_[K]; float dense[K], sparse[K]; int32_t rank[K], count = 0; int64_t ord[K];
    CHECK(krag_retrieve(ix, 1, vecs + 2 * DIM, q_terms, q_off, K, 3.0, 0.7, 0.3, KRAG_FUSION_REFERENCE, NULL, 0,
                        final_, dense, sparse, rank, ord, &count));
    for (int i = 0; i < count; ++i)
        printf("#%d node %lld  final %.6f  l2sq %.6f  bm25 %.6f (rank %d)\n", i, (long long)ord[i], final_[i], dense[i], sparse[i], (int)rank[i]);

    CHECK(krag_index_drop(ix));
    CHECK(krag_shutdown(ctx));
    return 0;
}
