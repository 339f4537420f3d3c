/*
 * TEST INFRASTRUCTURE — NOT PRODUCT CODE.
 *
 * Sequential CPU restatement of the C-SVC solver behind the reference's voxelwise cross-validation
 * (voxelselector.py:41-53: sklearn cross_val_score(SVC(kernel='precomputed')) -> libsvm's SMO).  The solver is a
 * THIRD-PARTY dependency of the reference (scikit-learn; here 1.9.0, sklearn/svm/src/libsvm/svm.cpp: Solver::Solve,
 * select_working_set, do_shrinking, be_shrunk, reconstruct_gradient, calculate_rho), restated from its published
 * algorithm (Fan, Chen, Lin: "Working set selection using second order information", JMLR 2005; LIBSVM guide section 5)
 * in the data structure the CUDA kernels use: everything lives by POSITION, `pm[pos]` is the index of the item at that
 * position in the unpermuted two-class sub-problem, and Q is never permuted.
 *
 * Parity status: PINNED against scikit-learn itself -- tests/test_oracle.py requires the iteration count (SVC.n_iter_),
 * rho (intercept_) and the dual coefficients of every problem to equal scikit-learn's, with and without shrinking.
 * The GPU solver (k_svm_cv, with and without shrinking) is tested against scikit-learn directly; this file lets the CPU
 * suite check the same restated algorithm without a GPU.
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#define SMO_TAU 1e-12
#define SMO_MAXN 64

static __thread int g_min_active, g_reconstructs;   /* of the last solve on this thread: did the heuristic do anything? */
static __thread int g_by_rows, g_by_cols, g_final_active;   /* reconstructions per loop order; active set at the end */

typedef struct {
    int n, active, unshrink;
    double C, eps;
    const float *Q;           /* [n][n], unpermuted: Q[a][b] = (float)(y_a y_b K_ab) */
    int pm[SMO_MAXN];         /* active_set: item at a position */
    double y[SMO_MAXN], alpha[SMO_MAXN], G[SMO_MAXN], Gbar[SMO_MAXN], QD[SMO_MAXN];
} smo_t;

static double q_at(const smo_t *s, int pi, int pk) { return (double)s->Q[s->pm[pi] * s->n + s->pm[pk]]; }
static int at_upper(const smo_t *s, int k) { return s->alpha[k] >= s->C; }
static int at_lower(const smo_t *s, int k) { return s->alpha[k] <= 0; }

/* second-order working set selection over the active positions; returns 1 when already optimal */
static int smo_select(const smo_t *s, int *oi, int *oj)
{
    double gmax = -INFINITY, gmax2 = -INFINITY, best = INFINITY;
    int i = -1, j = -1;
    for (int t = 0; t < s->active; t++) {            /* ">=": the last maximiser wins */
        if (s->y[t] > 0) {
            if (!at_upper(s, t) && -s->G[t] >= gmax) { gmax = -s->G[t]; i = t; }
        } else {
            if (!at_lower(s, t) && s->G[t] >= gmax) { gmax = s->G[t]; i = t; }
        }
    }
    for (int t = 0; t < s->active; t++) {
        double gd, quad, obj;
        if (s->y[t] > 0) {
            if (at_lower(s, t)) continue;
            gd = gmax + s->G[t];
            if (s->G[t] >= gmax2) gmax2 = s->G[t];
            if (!(gd > 0)) continue;
            quad = s->QD[i] + s->QD[t] - 2.0 * s->y[i] * q_at(s, i, t);
        } else {
            if (at_upper(s, t)) continue;
            gd = gmax - s->G[t];
            if (-s->G[t] >= gmax2) gmax2 = -s->G[t];
            if (!(gd > 0)) continue;
            quad = s->QD[i] + s->QD[t] + 2.0 * s->y[i] * q_at(s, i, t);
        }
        obj = quad > 0 ? -(gd * gd) / quad : -(gd * gd) / SMO_TAU;
        if (obj <= best) { best = obj; j = t; }     /* "<=": the last minimiser wins */
    }
    if (gmax + gmax2 < s->eps || j < 0) return 1;
    *oi = i;
    *oj = j;
    return 0;
}

/* G of the inactive positions from G_bar and the free active variables (both loop orders of libsvm add the free
 * variables in ascending position; they read opposite triangles of Q) */
static void smo_reconstruct(smo_t *s)
{
    int n = s->n, nr_free = 0;
    if (s->active == n) return;
    ++g_reconstructs;
    for (int k = s->active; k < n; k++) s->G[k] = s->Gbar[k] + (-1.0);
    for (int k = 0; k < s->active; k++) nr_free += !at_upper(s, k) && !at_lower(s, k);
    int by_rows = (long)nr_free * n > 2L * s->active * (n - s->active);
    if (by_rows) ++g_by_rows; else ++g_by_cols;
    for (int jj = 0; jj < s->active; jj++) {
        if (at_upper(s, jj) || at_lower(s, jj)) continue;
        for (int k = s->active; k < n; k++)
            s->G[k] += s->alpha[jj] * (by_rows ? q_at(s, k, jj) : q_at(s, jj, k));
    }
}

static void smo_swap(smo_t *s, int a, int b)
{
#define SW(arr, T) do { T t_ = s->arr[a]; s->arr[a] = s->arr[b]; s->arr[b] = t_; } while (0)
    SW(pm, int); SW(y, double); SW(alpha, double); SW(G, double); SW(Gbar, double); SW(QD, double);
#undef SW
}

static int smo_be_shrunk(const smo_t *s, int k, double g1, double g2)
{
    if (at_upper(s, k)) return s->y[k] > 0 ? (-s->G[k] > g1) : (-s->G[k] > g2);
    if (at_lower(s, k)) return s->y[k] > 0 ? (s->G[k] > g2) : (s->G[k] > g1);
    return 0;
}

static void smo_shrink(smo_t *s)
{
    double g1 = -INFINITY, g2 = -INFINITY;
    for (int k = 0; k < s->active; k++) {
        if (s->y[k] > 0) {
            if (!at_upper(s, k) && -s->G[k] >= g1) g1 = -s->G[k];
            if (!at_lower(s, k) && s->G[k] >= g2) g2 = s->G[k];
        } else {
            if (!at_upper(s, k) && -s->G[k] >= g2) g2 = -s->G[k];
            if (!at_lower(s, k) && s->G[k] >= g1) g1 = s->G[k];
        }
    }
    if (!s->unshrink && g1 + g2 <= s->eps * 10) {
        s->unshrink = 1;
        smo_reconstruct(s);
        s->active = s->n;
    }
    for (int k = 0; k < s->active; k++) {
        if (!smo_be_shrunk(s, k, g1, g2)) continue;
        s->active--;
        while (s->active > k) {
            if (!smo_be_shrunk(s, s->active, g1, g2)) {
                smo_swap(s, k, s->active);
                break;
            }
            s->active--;
        }
    }
    if (s->active < g_min_active) g_min_active = s->active;
}

/* the analytic two-variable step with libsvm's clipping order */
static void smo_step(double *ai, double *aj, double yi, double yj, double qdi, double qdj, double qij, double gi, double gj,
                     double C)
{
    if (yi != yj) {
        double quad = qdi + qdj + 2 * qij;
        if (quad <= 0) quad = SMO_TAU;
        double delta = (-gi - gj) / quad, diff = *ai - *aj;
        *ai += delta;
        *aj += delta;
        if (diff > 0) { if (*aj < 0) { *aj = 0; *ai = diff; } }
        else          { if (*ai < 0) { *ai = 0; *aj = -diff; } }
        if (diff > C - C) { if (*ai > C) { *ai = C; *aj = C - diff; } }
        else              { if (*aj > C) { *aj = C; *ai = C + diff; } }
    } else {
        double quad = qdi + qdj - 2 * qij;
        if (quad <= 0) quad = SMO_TAU;
        double delta = (gi - gj) / quad, sum = *ai + *aj;
        *ai -= delta;
        *aj += delta;
        if (sum > C) { if (*ai > C) { *ai = C; *aj = sum - C; } }
        else         { if (*aj < 0) { *aj = 0; *ai = sum; } }
        if (sum > C) { if (*aj > C) { *aj = C; *ai = sum - C; } }
        else         { if (*ai < 0) { *ai = 0; *aj = sum; } }
    }
}

/* Solve one two-class problem.  K: [E][E] float32 kernel; train_idx[n]: samples, the n_pos of class +1 first.
 * alpha_out[n] in the order of train_idx; returns the number of iterations, *rho_out = the offset. */
int oracle_svm_smo(const float *K, int E, const int *train_idx, int n, int n_pos, double C, double eps, int max_iter,
                   int shrinking, double *alpha_out, double *rho_out)
{
    if (n < 2 || n > SMO_MAXN || n_pos < 1 || n_pos >= n) return -1;
    smo_t s;
    float *Q = (float *)malloc(sizeof(float) * n * n);
    g_min_active = n;
    g_reconstructs = 0;
    g_by_rows = g_by_cols = 0;
    s.n = s.active = n;
    s.unshrink = 0;
    s.C = C;
    s.eps = eps;
    s.Q = Q;
    for (int a = 0; a < n; a++) {
        float ya = a < n_pos ? 1.f : -1.f;
        for (int b = 0; b < n; b++) Q[a * n + b] = ya * (b < n_pos ? 1.f : -1.f) * K[train_idx[a] * E + train_idx[b]];
        s.pm[a] = a;
        s.y[a] = ya;
        s.alpha[a] = 0;
        s.G[a] = -1.0;
        s.Gbar[a] = 0;
        s.QD[a] = (double)K[train_idx[a] * E + train_idx[a]];
    }
    int iter = 0, counter = (n < 1000 ? n : 1000) + 1;
    for (;;) {
        int i, j;
        if (max_iter >= 0 && iter >= max_iter) break;   /* scikit-learn: -1 = no limit, 0 = no iteration */
        if (--counter == 0) {
            counter = n < 1000 ? n : 1000;
            if (shrinking) smo_shrink(&s);
        }
        if (smo_select(&s, &i, &j)) {
            smo_reconstruct(&s);
            s.active = n;
            if (smo_select(&s, &i, &j)) break;
            counter = 1;
        }
        ++iter;
        double ai = s.alpha[i], aj = s.alpha[j];
        const double oi = ai, oj = aj;
        smo_step(&ai, &aj, s.y[i], s.y[j], s.QD[i], s.QD[j], q_at(&s, i, j), s.G[i], s.G[j], C);
        const double dai = ai - oi, daj = aj - oj;
        for (int k = 0; k < s.active; k++) s.G[k] += q_at(&s, i, k) * dai + q_at(&s, j, k) * daj;
        const int ui = oi >= C, uj = oj >= C;
        s.alpha[i] = ai;
        s.alpha[j] = aj;
        if (ui != (ai >= C))
            for (int k = 0; k < n; k++) s.Gbar[k] = ui ? s.Gbar[k] - C * q_at(&s, i, k) : s.Gbar[k] + C * q_at(&s, i, k);
        if (uj != (aj >= C))
            for (int k = 0; k < n; k++) s.Gbar[k] = uj ? s.Gbar[k] - C * q_at(&s, j, k) : s.Gbar[k] + C * q_at(&s, j, k);
    }
    /* offset: mean of y G over the free variables, else the midpoint of the bounds */
    double ub = INFINITY, lb = -INFINITY, sum_free = 0;
    int nr_free = 0;
    for (int k = 0; k < s.active; k++) {
        double yG = s.y[k] * s.G[k];
        if (at_upper(&s, k)) { if (s.y[k] < 0) ub = fmin(ub, yG); else lb = fmax(lb, yG); }
        else if (at_lower(&s, k)) { if (s.y[k] > 0) ub = fmin(ub, yG); else lb = fmax(lb, yG); }
        else { ++nr_free; sum_free += yG; }
    }
    *rho_out = nr_free > 0 ? sum_free / nr_free : (ub + lb) / 2;
    g_final_active = s.active;
    for (int k = 0; k < n; k++) alpha_out[s.pm[k]] = s.alpha[k];
    free(Q);
    return iter;
}

/* decision value of a held-out sample: sum_k alpha_k y_k K(test, k) - rho, support vectors in the order of train_idx */
double oracle_svm_decision(const float *K, int E, const int *train_idx, int n, int n_pos, const double *alpha, double rho,
                           int test)
{
    double sum = 0;
    for (int k = 0; k < n; k++)
        if (alpha[k] != 0) sum += alpha[k] * (k < n_pos ? 1.0 : -1.0) * (double)K[test * E + train_idx[k]];
    return sum - rho;
}

/* smallest active set and number of gradient reconstructions of the last oracle_svm_smo call on this thread */
void oracle_svm_last_stats(int *min_active, int *reconstructs)
{
    *min_active = g_min_active;
    *reconstructs = g_reconstructs;
}

/* of the last oracle_svm_smo call on this thread: gradient reconstructions that read Q by rows / by columns, and the
 * active set when the loop ended (below n when max_iter cut it while variables were shrunk) */
void oracle_svm_last_detail(int *by_rows, int *by_cols, int *final_active)
{
    *by_rows = g_by_rows;
    *by_cols = g_by_cols;
    *final_active = g_final_active;
}
