/*
 * mlp64_solver_oracle.c — CPU restatement of the float64 MLP classifier's full stochastic solver surface
 * (nn/neural_network/basemlp64.go): solver "adam" or "sgd" with momentum / Nesterov (SGDOptimizer64, :987-1039),
 * learning-rate schedules "constant" / "invscaling" / "adaptive" (:999-1023, :1053-1073), hidden activations relu /
 * logistic / identity / tanh (:78-148) and weight decay (:342-346).
 *
 * TEST INFRASTRUCTURE ONLY.  oracle/mlp64_oracle.c restates the Adam-only path and stays the pinned checker for it;
 * this file is a superset written beside it, and tests/test_mlp64_solver_oracle.py holds the two equal (bit for bit)
 * wherever their surfaces overlap, and holds this one to numpy transcripts and finite differences elsewhere.
 *
 * Quirks kept on purpose, as in the reference:
 *   - tanh's forward is tanh(−z) (:91) but its derivative is taken as 1 − a² (:135), the derivative of tanh(z): the
 *     data term of the gradient is negated in every layer below an odd number of tanh layers;
 *   - weight decay multiplies the whole packed vector, intercepts included, before every minibatch's forward pass;
 *   - the invscaling sample count t survives warm-start fits (initialize, which zeroes it, is skipped: :411-412, 502).
 * Sequential per output element, the reductions in the device's order (k ascending, rows ascending); built with
 * -ffp-contract=off.
 */
#include "../oracle/ctr_oracle.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>

enum { SOLVER_ADAM = 0, SOLVER_SGD = 1 };
enum { LR_CONSTANT = 0, LR_INVSCALING = 1, LR_ADAPTIVE = 2 };
enum { ACT_TANH = 3 };

/* same layout as ctr_mlp_options (include/ctr_b200.h) */
typedef struct {
    int32_t solver, lr_schedule, nesterov, reserved0;
    double power_t, momentum, weight_decay;
    double reserved[5];
} sol_opts;

/* the counter RNG of the project (ctr_oracle.c orc_mix64, engine.cu mix64): init and epoch shuffle */
static uint64_t mix64(uint32_t seed, uint32_t stream, uint64_t ctr) {
    uint64_t z = (((uint64_t)seed << 32) | stream) * 0x9E3779B97F4A7C15ull + ctr * 0xD1B54A32D192ED03ull
                 + 0x632BE59BD9B4E019ull;
    z ^= z >> 30; z *= 0xBF58476D1CE4E5B9ull;
    z ^= z >> 27; z *= 0x94D049BB133111EBull;
    z ^= z >> 31;
    return z;
}

long sol_nparams(const orc_mlp64_cfg* c) {
    long n = 0;
    for (int i = 0; i + 1 < c->n_layers; i++) n += (long)(1 + c->units[i]) * c->units[i + 1];
    return n;
}
static long layer_off(const orc_mlp64_cfg* c, int layer) {
    long n = 0;
    for (int i = 0; i < layer; i++) n += (long)(1 + c->units[i]) * c->units[i + 1];
    return n;
}

/* initialize :458-476: U[0,1)·sqrt(f/(fi+fo)) for every packed element; f = 2 for logistic, else 6 (tanh included) */
void sol_init(const orc_mlp64_cfg* c, double* params) {
    long pos = 0;
    for (int i = 0; i + 1 < c->n_layers; i++) {
        int fi = c->units[i], fo = c->units[i + 1];
        double bound = sqrt((c->hidden_act == ORC_MLP_LOGISTIC ? 2.0 : 6.0) / (double)(fi + fo));
        long end = pos + (long)(1 + fi) * fo;
        for (; pos < end; pos++) params[pos] = (double)(mix64(c->seed, 7, (uint64_t)pos) >> 11) * (1.0 / 9007199254740992.0) * bound;
    }
}

/* forwardPass :259-275; act[0] = X [n, units[0]] */
static void forward(const orc_mlp64_cfg* c, const double* params, double** act, long n) {
    int L = c->n_layers;
    for (int l = 0; l + 1 < L; l++) {
        int fi = c->units[l], fo = c->units[l + 1], last = (l + 1 == L - 1);
        const double* b = params + layer_off(c, l);
        const double* W = b + fo;
#pragma omp parallel for schedule(static)
        for (long r = 0; r < n; r++) {
            const double* a = act[l] + r * fi;
            for (int j = 0; j < fo; j++) {
                double z = 0.0;
                for (int k = 0; k < fi; k++) z += a[k] * W[(long)k * fo + j];
                z += b[j];                                                       /* addIntercepts64 :205 */
                if (last || c->hidden_act == ORC_MLP_LOGISTIC) z = 1.0 / (1.0 + exp(-z));   /* :82-88, :423-425 */
                else if (c->hidden_act == ORC_MLP_RELU) z = z < 0.0 ? 0.0 : z;      /* :96-104 */
                else if (c->hidden_act == ACT_TANH) z = tanh(-z);                  /* :88-94 */
                act[l + 1][r * fo + j] = z;
            }
        }
    }
}

typedef struct { double** act; double** del; } sol_ws;
static sol_ws ws_new(const orc_mlp64_cfg* c, long n) {
    sol_ws w;
    w.act = (double**)calloc(c->n_layers, sizeof(double*));
    w.del = (double**)calloc(c->n_layers, sizeof(double*));
    for (int l = 1; l < c->n_layers; l++) {
        w.act[l] = (double*)malloc(sizeof(double) * n * c->units[l]);
        w.del[l] = (double*)malloc(sizeof(double) * n * c->units[l]);
    }
    return w;
}
static void ws_free(const orc_mlp64_cfg* c, sol_ws w) {
    for (int l = 1; l < c->n_layers; l++) { free(w.act[l]); free(w.del[l]); }
    free(w.act); free(w.del);
}

/* backprop :340-406 after any weight decay: loss (binary_log_loss :180-195 + L2 :361) and packed gradients */
static double backprop(const orc_mlp64_cfg* c, const double* params, const double* X, const double* y, long n,
                       sol_ws ws, double* grads) {
    int L = c->n_layers, no = c->units[L - 1];
    ws.act[0] = (double*)X;
    forward(c, params, ws.act, n);
    const double hmin = nextafter(0.0, 1.0), hmax = nextafter(1.0, 0.0);
    double s = 0.0;
    for (long i = 0; i < n * no; i++) {
        double hv = ws.act[L - 1][i];
        ws.del[L - 1][i] = hv - y[i];                                            /* :373-381 */
        hv = hv < hmin ? hmin : (hv > hmax ? hmax : hv);
        s += -y[i] * log(hv) - (1.0 - y[i]) * log1p(-hv);
    }
    double sq = 0.0;                                                             /* sumCoefSquares :311-319 */
    for (int l = 0; l + 1 < L; l++) {
        const double* W = params + layer_off(c, l) + c->units[l + 1];
        long cnt = (long)c->units[l] * c->units[l + 1];
        for (long i = 0; i < cnt; i++) sq += W[i] * W[i];
    }
    double loss = s / (double)n + (0.5 * c->alpha) * sq / (double)n;
    for (int l = L - 2; l >= 0; l--) {
        int fi = c->units[l], fo = c->units[l + 1];
        const double* W = params + layer_off(c, l) + fo;
        double* gb = grads + layer_off(c, l);
        double* gW = gb + fo;
        const double* A = ws.act[l];
        const double* D = ws.del[l + 1];
#pragma omp parallel for schedule(static)
        for (int k = 0; k < fi; k++) {                                           /* computeLossGrad :322-331 */
            for (int j = 0; j < fo; j++) {
                double g = 0.0;
                for (long r = 0; r < n; r++) g += A[r * fi + k] * D[r * fo + j];
                gW[(long)k * fo + j] = g / (double)n + c->alpha / (double)n * W[(long)k * fo + j];
            }
        }
        for (int j = 0; j < fo; j++) {                                           /* matRowMean64 :213-226 */
            double m = 0.0;
            for (long r = 0; r < n; r++) m += D[r * fo + j];
            gb[j] = m / (double)n;
        }
        if (l >= 1) {                                                            /* :388-396 */
#pragma omp parallel for schedule(static)
            for (long r = 0; r < n; r++) {
                for (int k = 0; k < fi; k++) {
                    double d = 0.0;
                    for (int j = 0; j < fo; j++) d += D[r * fo + j] * W[(long)k * fo + j];
                    double z = A[r * fi + k];
                    if (c->hidden_act == ORC_MLP_RELU) { if (z == 0.0) d = 0.0; }          /* :140-148 */
                    else if (c->hidden_act == ORC_MLP_LOGISTIC) d *= z * (1.0 - z);        /* :124-131 */
                    else if (c->hidden_act == ACT_TANH) d *= 1.0 - z * z;                 /* :131-138 */
                    ws.del[l][r * fi + k] = d;
                }
            }
        }
    }
    return loss;
}

double sol_loss_grad(const orc_mlp64_cfg* c, const double* params, const double* X, const double* y, long n, double* grads) {
    sol_ws ws = ws_new(c, n);
    double loss = backprop(c, params, X, y, n, ws, grads);
    ws_free(c, ws);
    return loss;
}

void sol_predict(const orc_mlp64_cfg* c, const double* params, const double* X, long n, double* out) {
    sol_ws ws = ws_new(c, n);
    ws.act[0] = (double*)X;
    forward(c, params, ws.act, n);
    memcpy(out, ws.act[c->n_layers - 1], sizeof(double) * n * c->units[c->n_layers - 1]);
    ws_free(c, ws);
}

/* SGDOptimizer64.updateParams :1024-1039 */
void sol_sgd(const sol_opts* o, double lr, double* params, const double* grads, double* vel, long np) {
    for (long i = 0; i < np; i++) {
        double update = o->momentum * vel[i] - lr * grads[i];
        vel[i] = update;
        if (o->nesterov) params[i] += o->momentum * update - lr * grads[i];
        else params[i] += update;
    }
}

/* backprop :342-346 */
void sol_decay(double weight_decay, double* params, long np) {
    if (weight_decay > 0)
        for (long i = 0; i < np; i++) params[i] *= (1 - weight_decay);
}

/* AdamOptimizer64.updateParams :1075-1091, β powers advancing once per element; *calls = opt.t */
static void adam(const orc_mlp64_cfg* c, double lr_init, double* calls, double* b1t, double* b2t, double* params,
                 const double* grads, double* ms, double* vs, long np, double* lr) {
    if (*calls == 0) { memset(ms, 0, sizeof(double) * np); memset(vs, 0, sizeof(double) * np); *b1t = 1; *b2t = 1; }
    *calls += 1;
    for (long i = 0; i < np; i++) {
        double g = grads[i];
        ms[i] = c->beta1 * ms[i] + (1 - c->beta1) * g;
        vs[i] = c->beta2 * vs[i] + (1 - c->beta2) * g * g;
        *b1t *= c->beta1;
        *b2t *= c->beta2;
        *lr = lr_init * sqrt(1 - *b2t) / (1. - *b1t);
        params[i] += -*lr * ms[i] / (sqrt(vs[i]) + c->eps);
    }
}

/* fit → fitStochastic :484-567, :729-857 on parameters the caller initialised (or kept, for a warm start).  *t is
 * BaseMultilayerPerceptron64.t in and out (the caller zeroes it after a cold initialise).  lr_curve (may be NULL)
 * receives the optimizer's learning rate after every epoch end (sgd: the one the next epoch uses; adam: the
 * base rate).  Returns NIter. */
int sol_fit(const orc_mlp64_cfg* c, const sol_opts* o, double* params, const double* X, const double* y, long n,
            double* loss_curve, double* lr_curve, double* t) {
    int L = c->n_layers, nin = c->units[0], no = c->units[L - 1];
    long np = sol_nparams(c);
    long bs = c->batch;
    if (bs <= 0) bs = n < 200 ? n : 200; else if (bs > n) bs = n;                /* :517-527 */
    sol_ws ws = ws_new(c, bs);
    double* grads = (double*)malloc(sizeof(double) * np);
    double* ms = (double*)calloc(np, sizeof(double));                            /* a fresh optimizer per fit :731-752 */
    double* vs = (double*)calloc(np, sizeof(double));
    double* Xb = (double*)malloc(sizeof(double) * bs * nin);
    double* yb = (double*)malloc(sizeof(double) * bs * no);
    long* idx = (long*)malloc(sizeof(long) * n);
    for (long i = 0; i < n; i++) idx[i] = i;
    const int sgd = o->solver == SOLVER_SGD;
    double lr = c->lr_init, lr_init = c->lr_init, calls = 0, b1t = 1, b2t = 1;
    double best = INFINITY;
    int no_improve = 0, it;
    for (it = 0; it < c->max_iter;) {
        if (c->shuffle) {                                                        /* rand.Shuffle :788, from the top */
            for (long i = n - 1; i > 0; i--) {
                long j = (long)(mix64(c->seed, 100 + (uint32_t)it, (uint64_t)i) % (uint64_t)(i + 1));
                long tmp = idx[i]; idx[i] = idx[j]; idx[j] = tmp;
            }
        }
        double acc = 0;
        for (long b0 = 0; b0 < n; b0 += bs) {                                    /* :791-808 */
            long m = (b0 + bs > n ? n : b0 + bs) - b0;
            for (long r = 0; r < m; r++) {
                memcpy(Xb + r * nin, X + idx[b0 + r] * nin, sizeof(double) * nin);
                memcpy(yb + r * no, y + idx[b0 + r] * no, sizeof(double) * no);
            }
            sol_decay(o->weight_decay, params, np);
            acc += backprop(c, params, Xb, yb, m, ws, grads) * (double)m;
            if (sgd) sol_sgd(o, lr, params, grads, ms, np);
            else adam(c, lr_init, &calls, &b1t, &b2t, params, grads, ms, vs, np, &lr);
        }
        it++;
        double loss = acc / (double)n;                                           /* :811-812 */
        *t += (double)n;                                                         /* :814 */
        if (loss_curve) loss_curve[it - 1] = loss;
        if (loss > best - c->tol) no_improve++; else no_improve = 0;             /* updateNoImprovementCount :884-894 */
        if (loss < best) best = loss;
        if (sgd && o->lr_schedule == LR_INVSCALING) lr = c->lr_init / pow(*t + 1, o->power_t);   /* iterationEnds :999-1003 */
        int stop = 0;
        if (no_improve > c->n_iter_no_change) {                                  /* :826-840 */
            if (o->lr_schedule != LR_ADAPTIVE) stop = 1;                         /* triggerStopping :1005-1011, :1054-1060 */
            else if (lr <= 1e-6) stop = 1;                                       /* :1012-1017, :1061-1066 */
            else { if (sgd) lr *= .8; else lr_init *= .8; no_improve = 0; }      /* :1018, :1067 */
        }
        if (lr_curve) lr_curve[it - 1] = sgd ? lr : lr_init;
        if (stop) break;
    }
    free(idx); free(Xb); free(yb); free(ms); free(vs); free(grads);
    ws_free(c, ws);
    return it;
}
