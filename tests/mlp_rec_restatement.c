/* mlp_rec_restatement.c — the float64 MLP's output-layer logit restated on the CPU for
 * tests/test_gpu_mlp64_recommend.py: for each input row, every layer walks
 *   z = 0; z = fma(a[k], W[k, j], z) for k ascending; z = z + b[j]
 * (the chain k_mlp64_layer and the recommendation kernels run, one DFMA per term), then the hidden activation
 * (relu, logistic 1 / (1 + exp(-z)), identity, tanh(-z)); the output layer keeps z, the logit.  Parameters use the
 * packed layout of ctr_mlp_get_params: per layer [intercepts (fo) | coefs (fi x fo row-major)].
 * Build: gcc -O2 -std=c99 -ffp-contract=off -shared -fPIC -o lib.so mlp_rec_restatement.c -lm */
#include <math.h>
#include <stdlib.h>

enum { ACT_RELU = 0, ACT_LOGISTIC = 1, ACT_IDENTITY = 2, ACT_TANH = 3 };

/* X [n, units[0]] float64 rows, logits [n] */
void rec_logits(const double* params, int n_layers, const int* units, int act, const double* X, long n, double* logits) {
    int wmax = 0;
    for (int l = 0; l < n_layers; l++) if (units[l] > wmax) wmax = units[l];
    double* a = malloc(sizeof(double) * (size_t)wmax);
    double* o = malloc(sizeof(double) * (size_t)wmax);
    for (long r = 0; r < n; r++) {
        for (int k = 0; k < units[0]; k++) a[k] = X[r * units[0] + k];
        long off = 0;
        for (int l = 0; l + 1 < n_layers; l++) {
            const int fi = units[l], fo = units[l + 1];
            const double* b = params + off;
            const double* W = b + fo;
            const int last = l + 2 == n_layers;
            for (int j = 0; j < fo; j++) {
                double z = 0.0;
                for (int k = 0; k < fi; k++) z = fma(a[k], W[(long)k * fo + j], z);
                z = z + b[j];
                if (!last) {
                    if (act == ACT_LOGISTIC) z = 1.0 / (1.0 + exp(-z));
                    else if (act == ACT_RELU) z = z < 0.0 ? 0.0 : z;
                    else if (act == ACT_TANH) z = tanh(-z);
                }
                o[j] = z;
            }
            for (int j = 0; j < fo; j++) a[j] = o[j];
            off += (long)(1 + fi) * fo;
        }
        logits[r] = a[0];
    }
    free(a);
    free(o);
}
