/* knn_oracle.c — CPU restatement of search.Searcher (auxten/go-ctr feature/embedding/search/search.go:66-134),
 * the checker of ctr_knn_search.  TEST INFRASTRUCTURE ONLY (see ctr_oracle.h); built with -ffp-contract=off, as Go on
 * amd64 never fuses a multiply and an add.
 *
 *   embutil.Norm      emb/embutil/embutil.go:21-27      sqrt(sum v*v), sequential float64
 *   searchutil.Cosine search/searchutil/searchutil.go:17-26   0 if a norm is 0, else dot / n1 / n2
 *   Searcher.Search   search.go:94-134                  low threshold + bubble insertion, literally
 *
 * Input: the float32 table [N, D] (widened to float64, as emb.Load's vectors would be after a float32 round trip),
 * float64 queries [nq, D] and per query a row to ignore (-1: none; SearchInternal ignores the query's own word,
 * search.go:66-80).  Output per query: k (row, similarity) slots in the reference's order; empty slots are row -1,
 * similarity 0 (a zero Neighbor{}), and count = slots holding a word. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

double orc_knn_norm(const double* v, int D) {
    double n = 0;
    for (int d = 0; d < D; d++) n += v[d] * v[d];                  /* embutil.go:23-25 */
    return sqrt(n);
}

double orc_knn_cosine(const double* v1, const double* v2, double n1, double n2, int D) {
    if (n1 == 0 || n2 == 0) return 0;                               /* searchutil.go:18-20 */
    double dot = 0;
    for (int d = 0; d < D; d++) dot += v1[d] * v2[d];               /* :21-24 */
    return dot / n1 / n2;                                           /* :25 */
}

void orc_knn_search(const float* table, long N, int D, const double* queries, const int32_t* ignore, long nq, int k,
                    int32_t* out_rows, double* out_sim, int32_t* out_count) {
    double* nv = (double*)malloc(sizeof(double) * (size_t)(N > 0 ? N : 1));
    double* row = (double*)malloc(sizeof(double) * (size_t)N * D + 8);
    for (long i = 0; i < N; i++) {                                  /* Embedding.Norm of every item, once */
        for (int d = 0; d < D; d++) row[(size_t)i * D + d] = (double)table[(size_t)i * D + d];
        nv[i] = orc_knn_norm(row + (size_t)i * D, D);
    }
#pragma omp parallel for schedule(dynamic)
    for (long q = 0; q < nq; q++) {
        const double* qv = queries + (size_t)q * D;
        const double qn = orc_knn_norm(qv, D);
        int32_t* nr = out_rows + (size_t)q * k;                     /* neighbors := make(Neighbors, k), :95 */
        double* ns = out_sim + (size_t)q * k;
        for (int i = 0; i < k; i++) { nr[i] = -1; ns[i] = 0; }
        double low = 0;                                             /* :104 */
        for (long it = 0; it < N; it++) {
            if (ignore && ignore[q] == it) continue;                /* :107-110 */
            const double score = orc_knn_cosine(qv, row + (size_t)it * D, qn, nv[it], D);
            if (score > low) {                                      /* :114 */
                int32_t tr = (int32_t)it; double ts = score;
                for (int i = 0; i < k; i++) {                       /* bubble up, :117-122 */
                    if (ts > ns[i]) {
                        int32_t r = nr[i]; double s = ns[i];
                        nr[i] = tr; ns[i] = ts; tr = r; ts = s;
                    }
                }
                low = ns[k - 1];                                    /* :124 */
            }
        }
        int c = 0;
        while (c < k && nr[c] != -1) c++;
        out_count[q] = c;
    }
    free(row); free(nv);
}
