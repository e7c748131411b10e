/*
 * mlp64_reg_oracle.c — CPU restatement of the float64 MLP regressor (nn/neural_network/multilayer_perceptron.go:9-71
 * MLPRegressor over BaseMultilayerPerceptron64): fit(X, Y, false) on dense targets Y [n, no] (:46-50), the output kind
 * a cold initialise takes from all targets (basemlp64.go:502-511 → initialize :416-430), square_loss (:152-161) or
 * log_loss (:162-178) or binary_log_loss (:180-195) with delta h − y (:373-381), Predict (the raw output layer,
 * :53-62) and Score (r2Score64, :1116-1141).  The solver loop (minibatches, shuffle, adam / sgd, schedules, weight
 * decay, stopping rules, the t carry) is the one of tests/mlp64_class_oracle.c and tests/mlp64_solver_oracle.c.
 *
 * TEST INFRASTRUCTURE ONLY.  The output kind is passed explicitly (REG_OUT_*, as CTR_MLP_OUT_*); reg_out_kind decides
 * it from the targets as the reference does.  Sequential per output element, the reductions in the reference's order;
 * built with -ffp-contract=off.
 */
#include "../oracle/ctr_oracle.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>

enum { SOLVER_SGD = 1 };
enum { LR_INVSCALING = 1, LR_ADAPTIVE = 2 };
enum { ACT_TANH = 3 };
enum { REG_OUT_IDENTITY = 0, REG_OUT_LOGISTIC = 1, REG_OUT_SOFTMAX = 2 };

typedef struct {                 /* ctr_mlp_options (include/ctr_b200.h) */
    int32_t solver, lr_schedule, nesterov, reserved0;
    double power_t, momentum, weight_decay;
    double reserved[5];
} reg_opts;

static uint64_t mix64(uint32_t seed, uint32_t stream, uint64_t ctr) {
    uint64_t z = (((uint64_t)seed << 32) | stream) * 0x9E3779B97F4A7C15ull + ctr * 0xD1B54A32D192ED03ull
                 + 0x632BE59BD9B4E019ull;
    z ^= z >> 30; z *= 0xBF58476D1CE4E5B9ull;
    z ^= z >> 27; z *= 0x94D049BB133111EBull;
    z ^= z >> 31;
    return z;
}

/* fit :502-511: some target not 0 or 1 → identity; else one column → logistic, more → softmax */
int reg_out_kind(const float* y, long n, int no) {
    for (long i = 0; i < n * no; i++)
        if (y[i] != 0.0f && y[i] != 1.0f) return REG_OUT_IDENTITY;
    return no > 1 ? REG_OUT_SOFTMAX : REG_OUT_LOGISTIC;
}

long reg_nparams(const orc_mlp64_cfg* c) {
    long n = 0;
    for (int i = 0; i + 1 < c->n_layers; i++) n += (long)(1 + c->units[i]) * c->units[i + 1];
    return n;
}
static long layer_off(const orc_mlp64_cfg* c, int layer) {
    long n = 0;
    for (int i = 0; i < layer; i++) n += (long)(1 + c->units[i]) * c->units[i + 1];
    return n;
}

/* initialize :458-476 */
void reg_init(const orc_mlp64_cfg* c, double* params) {
    long pos = 0;
    for (int i = 0; i + 1 < c->n_layers; i++) {
        int fi = c->units[i], fo = c->units[i + 1];
        double bound = sqrt((c->hidden_act == ORC_MLP_LOGISTIC ? 2.0 : 6.0) / (double)(fi + fo));
        long end = pos + (long)(1 + fi) * fo;
        for (; pos < end; pos++) params[pos] = (double)(mix64(c->seed, 7, (uint64_t)pos) >> 11) * (1.0 / 9007199254740992.0) * bound;
    }
}

/* forwardPass :259-275; act[0] = X; the output layer by kind */
static void forward(const orc_mlp64_cfg* c, int kind, const double* params, double** act, long n) {
    int L = c->n_layers, no = c->units[L - 1];
    for (int l = 0; l + 1 < L; l++) {
        int fi = c->units[l], fo = c->units[l + 1], last = (l + 1 == L - 1);
        const double* b = params + layer_off(c, l);
        const double* W = b + fo;
        int act_kind = last ? (kind == REG_OUT_LOGISTIC ? ORC_MLP_LOGISTIC : ORC_MLP_IDENTITY) : c->hidden_act;
        for (long r = 0; r < n; r++) {
            const double* a = act[l] + r * fi;
            for (int j = 0; j < fo; j++) {
                double z = 0.0;
                for (int k = 0; k < fi; k++) z += a[k] * W[(long)k * fo + j];
                z += b[j];
                if (act_kind == ORC_MLP_LOGISTIC) z = 1.0 / (1.0 + exp(-z));
                else if (act_kind == ORC_MLP_RELU) z = z < 0.0 ? 0.0 : z;
                else if (act_kind == ACT_TANH) z = tanh(-z);
                act[l + 1][r * fo + j] = z;
            }
        }
    }
    if (kind == REG_OUT_SOFTMAX)
        for (long r = 0; r < n; r++) {                                           /* softmax :104-117 */
            double* z = act[L - 1] + r * no;
            double sum = 0.0;
            for (int j = 0; j < no; j++) { z[j] = exp(z[j]); sum += z[j]; }
            for (int j = 0; j < no; j++) z[j] /= sum;
        }
}

typedef struct { double** act; double** del; } reg_ws;
static reg_ws ws_new(const orc_mlp64_cfg* c, long n) {
    reg_ws w;
    w.act = (double**)calloc(c->n_layers, sizeof(double*));
    w.del = (double**)calloc(c->n_layers, sizeof(double*));
    for (int l = 1; l < c->n_layers; l++) {
        w.act[l] = (double*)malloc(sizeof(double) * n * c->units[l]);
        w.del[l] = (double*)malloc(sizeof(double) * n * c->units[l]);
    }
    return w;
}
static void ws_free(const orc_mlp64_cfg* c, reg_ws w) {
    for (int l = 1; l < c->n_layers; l++) { free(w.act[l]); free(w.del[l]); }
    free(w.act); free(w.del);
}

/* backprop :340-406: the loss of the kind + L2 (:361); delta h − y (:373-381); computeLossGrad :322-331 */
static double backprop(const orc_mlp64_cfg* c, int kind, const double* params, const double* X, const double* y, long n,
                       reg_ws ws, double* grads) {
    int L = c->n_layers, no = c->units[L - 1];
    ws.act[0] = (double*)X;
    forward(c, kind, params, ws.act, n);
    const double hmin = nextafter(0.0, 1.0), hmax = nextafter(1.0, 0.0);
    double s = 0.0;
    for (long i = 0; i < n * no; i++) {
        double hv = ws.act[L - 1][i];
        double e = hv - y[i];
        ws.del[L - 1][i] = e;
        if (kind == REG_OUT_IDENTITY) { s += e * e; continue; }                 /* square_loss :152-161 */
        hv = hv < hmin ? hmin : (hv > hmax ? hmax : hv);
        if (kind == REG_OUT_SOFTMAX) { if (y[i] != 0) s += -y[i] * log(hv); }  /* log_loss :162-178 */
        else s += -y[i] * log(hv) - (1.0 - y[i]) * log1p(-hv);                  /* binary_log_loss :180-195 */
    }
    double sq = 0.0;
    for (int l = 0; l + 1 < L; l++) {
        const double* W = params + layer_off(c, l) + c->units[l + 1];
        long cnt = (long)c->units[l] * c->units[l + 1];
        for (long i = 0; i < cnt; i++) sq += W[i] * W[i];
    }
    double data = kind == REG_OUT_IDENTITY ? s / 2 / (double)n : s / (double)n;
    double loss = data + (0.5 * c->alpha) * sq / (double)n;
    for (int l = L - 2; l >= 0; l--) {
        int fi = c->units[l], fo = c->units[l + 1];
        const double* W = params + layer_off(c, l) + fo;
        double* gb = grads + layer_off(c, l);
        double* gW = gb + fo;
        const double* A = ws.act[l];
        const double* D = ws.del[l + 1];
        for (int k = 0; k < fi; k++)
            for (int j = 0; j < fo; j++) {
                double g = 0.0;
                for (long r = 0; r < n; r++) g += A[r * fi + k] * D[r * fo + j];
                gW[(long)k * fo + j] = g / (double)n + c->alpha / (double)n * W[(long)k * fo + j];
            }
        for (int j = 0; j < fo; j++) {
            double m = 0.0;
            for (long r = 0; r < n; r++) m += D[r * fo + j];
            gb[j] = m / (double)n;
        }
        if (l >= 1)
            for (long r = 0; r < n; r++)
                for (int k = 0; k < fi; k++) {
                    double d = 0.0;
                    for (int j = 0; j < fo; j++) d += D[r * fo + j] * W[(long)k * fo + j];
                    double z = A[r * fi + k];
                    if (c->hidden_act == ORC_MLP_RELU) { if (z == 0.0) d = 0.0; }
                    else if (c->hidden_act == ORC_MLP_LOGISTIC) d *= z * (1.0 - z);
                    else if (c->hidden_act == ACT_TANH) d *= 1.0 - z * z;
                    ws.del[l][r * fi + k] = d;
                }
    }
    return loss;
}

double reg_loss_grad(const orc_mlp64_cfg* c, int kind, const double* params, const double* X, const double* y, long n, double* grads) {
    reg_ws ws = ws_new(c, n);
    double loss = backprop(c, kind, params, X, y, n, ws, grads);
    ws_free(c, ws);
    return loss;
}

/* Predict :53-62 → predictProbas: [n, units[L-1]] */
void reg_predict(const orc_mlp64_cfg* c, int kind, const double* params, const double* X, long n, double* out) {
    reg_ws ws = ws_new(c, n);
    ws.act[0] = (double*)X;
    forward(c, kind, params, ws.act, n);
    memcpy(out, ws.act[c->n_layers - 1], sizeof(double) * n * c->units[c->n_layers - 1]);
    ws_free(c, ws);
}

/* r2Score64 :1116-1141 over yt, yp [n, no]; *bad = the first column whose den is 0 (the reference panics), or −1 */
double reg_r2(const double* yt, const double* yp, long n, int no, long* bad) {
    double r2acc = 0.0;
    *bad = -1;
    for (int c = 0; c < no; c++) {
        double avg = 0.0, num = 0.0, den = 0.0;
        for (long r = 0; r < n; r++) avg += yt[r * no + c];
        avg /= (double)n;
        for (long r = 0; r < n; r++) {
            double t = yp[r * no + c] - yt[r * no + c];
            num += t * t;
            t = yt[r * no + c] - avg;
            den += t * t;
        }
        if (den == 0 && *bad < 0) *bad = c;
        r2acc += 1 - num / den;
    }
    return r2acc / (double)no;
}

/* fitStochastic :729-857 on Y [n, units[L-1]], in place on params; as cls_fit of mlp64_class_oracle.c */
int reg_fit(const orc_mlp64_cfg* c, int kind, const reg_opts* o, double* params, const double* X, const double* y, long n,
            double* loss_curve, double* t) {
    int L = c->n_layers, nin = c->units[0], no = c->units[L - 1];
    long np = reg_nparams(c);
    long bs = c->batch;
    if (bs <= 0) bs = n < 200 ? n : 200; else if (bs > n) bs = n;
    reg_ws ws = ws_new(c, bs);
    double* grads = (double*)malloc(sizeof(double) * np);
    double* ms = (double*)calloc(np, sizeof(double));
    double* vs = (double*)calloc(np, sizeof(double));
    double* Xb = (double*)malloc(sizeof(double) * bs * nin);
    double* yb = (double*)malloc(sizeof(double) * bs * no);
    long* idx = (long*)malloc(sizeof(long) * n);
    for (long i = 0; i < n; i++) idx[i] = i;
    const int sgd = o->solver == SOLVER_SGD;
    double lr = c->lr_init, lr_init = c->lr_init, b1t = 1, b2t = 1;
    double best = INFINITY;
    int no_improve = 0, it;
    for (it = 0; it < c->max_iter;) {
        if (c->shuffle)
            for (long i = n - 1; i > 0; i--) {
                long j = (long)(mix64(c->seed, 100 + (uint32_t)it, (uint64_t)i) % (uint64_t)(i + 1));
                long tmp = idx[i]; idx[i] = idx[j]; idx[j] = tmp;
            }
        double acc = 0;
        for (long b0 = 0; b0 < n; b0 += bs) {
            long m = (b0 + bs > n ? n : b0 + bs) - b0;
            for (long r = 0; r < m; r++) {
                memcpy(Xb + r * nin, X + idx[b0 + r] * nin, sizeof(double) * nin);
                memcpy(yb + r * no, y + idx[b0 + r] * no, sizeof(double) * no);
            }
            if (o->weight_decay > 0)
                for (long i = 0; i < np; i++) params[i] *= (1 - o->weight_decay);
            acc += backprop(c, kind, params, Xb, yb, m, ws, grads) * (double)m;
            for (long i = 0; i < np; i++) {
                double g = grads[i];
                if (sgd) {
                    double update = o->momentum * ms[i] - lr * g;
                    ms[i] = update;
                    params[i] += o->nesterov ? o->momentum * update - lr * g : update;
                } else {
                    ms[i] = c->beta1 * ms[i] + (1 - c->beta1) * g;
                    vs[i] = c->beta2 * vs[i] + (1 - c->beta2) * g * g;
                    b1t *= c->beta1;
                    b2t *= c->beta2;
                    lr = lr_init * sqrt(1 - b2t) / (1. - b1t);
                    params[i] += -lr * ms[i] / (sqrt(vs[i]) + c->eps);
                }
            }
        }
        it++;
        double loss = acc / (double)n;
        *t += (double)n;
        if (loss_curve) loss_curve[it - 1] = loss;
        if (loss > best - c->tol) no_improve++; else no_improve = 0;
        if (loss < best) best = loss;
        if (sgd && o->lr_schedule == LR_INVSCALING) lr = c->lr_init / pow(*t + 1, o->power_t);
        int stop = 0;
        if (no_improve > c->n_iter_no_change) {
            if (o->lr_schedule != LR_ADAPTIVE) stop = 1;
            else if (lr <= 1e-6) stop = 1;
            else { if (sgd) lr *= .8; else lr_init *= .8; no_improve = 0; }
        }
        if (stop) break;
    }
    free(idx); free(Xb); free(yb); free(ms); free(vs); free(grads);
    ws_free(c, ws);
    return it;
}
