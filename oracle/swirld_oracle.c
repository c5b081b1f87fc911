/*
 * swirld_oracle.c -- CPU restatement of py-swirld's consensus hot path.
 *
 * TEST INFRASTRUCTURE.  This file is the parity oracle for the CUDA engine in
 * py-swirld_b200/csrc/.  Only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs may load it; the product path never
 * does (it fails loudly when the CUDA library is missing).
 *
 * Parity status: PINNED.  tests/test_oracle_golden.py checks this code against
 * fixtures under tests/golden/ that oracle/make_golden.py produced by running
 * the unmodified py-swirld swirld.py (imported, never copied) on the same
 * traces and call schedules.
 *
 * The restatement is LITERAL on purpose: it follows the reference statement by
 * statement in index space (event id = arrival index, member id = 0..M-1,
 * "absent dict key" = -1) and keeps the reference's O(M^2)-per-event loops, its
 * float thresholds, its height-based `higher`, its vote dictionary and its
 * insertion-ordered witness dicts.  None of the engine's reformulations
 * (index compares, bit matrices, per-chain cut-offs) appear here, so that the
 * two can disagree.
 *
 * Reference lines are cited as swirld.py:<line> (= py-swirld's swirld.py).
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define OR_ERR_INDEX   (-2)  /* times[(n+1)//2] IndexError, swirld.py:305 */
#define OR_ERR_ARG     (-1)
#define OR_ERR_KEY     (-3)  /* votes[w][x] KeyError, swirld.py:260 */

/* Branch counters (or_coverage): how often a run took each rarely taken branch,
 * so that a test can assert that its trace reaches the branch it is meant to
 * test.  Counting never changes a result. */
enum {
    OR_COV_COIN_VOTES,       /* :272 votes cast by the coin */
    OR_COV_COIN_ONES,        /* ... of which the coin said 1 */
    OR_COV_COIN_SUPER,       /* :268-269 supermajority vote in a coin round */
    OR_COV_DECIDE_AFTER_C,   /* :262-264 decisions at r_ - r > C */
    OR_COV_DECISIONS,        /* :262-264 all decisions */
    OR_COV_MAJORITY_EMPTY,   /* :260 majority() over an empty s */
    OR_COV_MEDIAN_ODD,       /* :305 median over an odd number of times (the two middle-and-above entries) */
    OR_COV_MEDIAN_EVEN,      /* :305 median over an even number of times (one entry, twice) */
    OR_COV_SINGLE_SEER,      /* :305 IndexError: one time only */
    OR_COV_TIED,             /* :306 adjacent events of a round's final with equal consensus time */
    OR_NCOV
};

typedef struct {
    uint64_t *keys;   /* (y << 32 | x) + 1, 0 = empty */
    uint8_t  *vals;
    size_t cap, cnt;
} votemap;

typedef struct {
    int M, C;
    int64_t *stake;
    int64_t tot_stake;
    double min_s;                 /* swirld.py:44  2 * tot_stake / 3 */
    /* events (swirld.py:30 Event(d p t c s), 48 hg, 68 height) */
    int n, cap;
    int32_t *p0, *p1, *creator, *height;
    double *t;
    uint8_t *sig;                 /* n x 64 */
    /* swirld.py:72 can_see: n x M, -1 = key absent */
    int32_t *can_see;
    int32_t *round;               /* swirld.py:50 */
    int8_t *famous;               /* swirld.py:63: -1 no entry, 0 False, 1 True */
    uint8_t *tbd;                 /* swirld.py:52 */
    int32_t *idx;                 /* swirld.py:55 */
    int32_t *transactions;        /* swirld.py:54 */
    int n_tx;
    /* swirld.py:61 witnesses: per round an insertion-ordered dict member->event */
    int rcap, max_r;              /* max_r = max(self.witnesses), -1 if empty */
    int32_t *wt;                  /* rcap x M, -1 absent */
    int32_t *wt_order;            /* rcap x M: members in insertion order */
    int32_t *wt_cnt;              /* rcap */
    uint8_t *consensus;           /* swirld.py:57, per round */
    votemap votes;                /* swirld.py:59 */
    /* scratch */
    int64_t *hits;
    int32_t *queue;
    uint8_t *mark;
    int64_t cov[OR_NCOV];         /* branch counters, see OR_COV_* */
} oracle;

/* ---------------------------------------------------------------- votes */
static void vm_init(votemap *m) {
    m->cap = 1 << 16; m->cnt = 0;
    m->keys = (uint64_t *)calloc(m->cap, sizeof(uint64_t));
    m->vals = (uint8_t *)calloc(m->cap, 1);
}
static size_t vm_slot(const votemap *m, uint64_t k) {
    uint64_t h = k * 0x9E3779B97F4A7C15ull;
    size_t i = (size_t)(h >> 17) & (m->cap - 1);
    while (m->keys[i] && m->keys[i] != k) i = (i + 1) & (m->cap - 1);
    return i;
}
static void vm_put(votemap *m, uint32_t y, uint32_t x, int v);
static void vm_grow(votemap *m) {
    votemap o = *m;
    m->cap = o.cap * 2; m->cnt = 0;
    m->keys = (uint64_t *)calloc(m->cap, sizeof(uint64_t));
    m->vals = (uint8_t *)calloc(m->cap, 1);
    for (size_t i = 0; i < o.cap; i++)
        if (o.keys[i]) {
            size_t s = vm_slot(m, o.keys[i]);
            m->keys[s] = o.keys[i]; m->vals[s] = o.vals[i]; m->cnt++;
        }
    free(o.keys); free(o.vals);
}
static void vm_put(votemap *m, uint32_t y, uint32_t x, int v) {
    uint64_t k = (((uint64_t)y << 32) | x) + 1;
    if ((m->cnt + 1) * 2 > m->cap) vm_grow(m);
    size_t s = vm_slot(m, k);
    if (!m->keys[s]) { m->keys[s] = k; m->cnt++; }
    m->vals[s] = (uint8_t)v;
}
static int vm_get(const votemap *m, uint32_t y, uint32_t x) {
    uint64_t k = (((uint64_t)y << 32) | x) + 1;
    size_t s = vm_slot(m, k);
    return m->keys[s] ? m->vals[s] : -1;
}

/* ---------------------------------------------------------------- life cycle */
void *or_create(int M, const int64_t *stake, int coin_period) {
    if (M < 1 || coin_period < 1) return NULL;
    oracle *o = (oracle *)calloc(1, sizeof(oracle));
    o->M = M; o->C = coin_period;
    o->stake = (int64_t *)malloc(sizeof(int64_t) * M);
    for (int c = 0; c < M; c++) {
        o->stake[c] = stake ? stake[c] : 1;
        o->tot_stake += o->stake[c];                 /* swirld.py:43 */
    }
    o->min_s = (double)(2 * o->tot_stake) / 3.0;     /* swirld.py:44 */
    o->max_r = -1;
    vm_init(&o->votes);
    o->hits = (int64_t *)malloc(sizeof(int64_t) * M);
    return o;
}

void or_destroy(void *h) {
    oracle *o = (oracle *)h;
    if (!o) return;
    free(o->stake); free(o->p0); free(o->p1); free(o->creator); free(o->height);
    free(o->t); free(o->sig); free(o->can_see); free(o->round); free(o->famous);
    free(o->tbd); free(o->idx); free(o->transactions); free(o->wt);
    free(o->wt_order); free(o->wt_cnt); free(o->consensus);
    free(o->votes.keys); free(o->votes.vals); free(o->hits); free(o->queue);
    free(o->mark); free(o);
}

static void grow_events(oracle *o, int need) {
    if (need <= o->cap) return;
    int cap = o->cap ? o->cap : 1024;
    while (cap < need) cap *= 2;
    size_t M = (size_t)o->M;
    o->p0 = (int32_t *)realloc(o->p0, sizeof(int32_t) * cap);
    o->p1 = (int32_t *)realloc(o->p1, sizeof(int32_t) * cap);
    o->creator = (int32_t *)realloc(o->creator, sizeof(int32_t) * cap);
    o->height = (int32_t *)realloc(o->height, sizeof(int32_t) * cap);
    o->t = (double *)realloc(o->t, sizeof(double) * cap);
    o->sig = (uint8_t *)realloc(o->sig, (size_t)64 * cap);
    o->can_see = (int32_t *)realloc(o->can_see, sizeof(int32_t) * M * cap);
    o->round = (int32_t *)realloc(o->round, sizeof(int32_t) * cap);
    o->famous = (int8_t *)realloc(o->famous, cap);
    o->tbd = (uint8_t *)realloc(o->tbd, cap);
    o->idx = (int32_t *)realloc(o->idx, sizeof(int32_t) * cap);
    o->transactions = (int32_t *)realloc(o->transactions, sizeof(int32_t) * cap);
    o->queue = (int32_t *)realloc(o->queue, sizeof(int32_t) * cap);
    o->mark = (uint8_t *)realloc(o->mark, cap);
    for (int i = o->cap; i < cap; i++) {
        o->round[i] = -1; o->famous[i] = -1; o->tbd[i] = 0; o->idx[i] = -1; o->mark[i] = 0;
    }
    o->cap = cap;
}

static void grow_rounds(oracle *o, int r) {
    if (r < o->rcap) return;
    int cap = o->rcap ? o->rcap : 64;
    while (cap <= r) cap *= 2;
    size_t M = (size_t)o->M;
    o->wt = (int32_t *)realloc(o->wt, sizeof(int32_t) * M * cap);
    o->wt_order = (int32_t *)realloc(o->wt_order, sizeof(int32_t) * M * cap);
    o->wt_cnt = (int32_t *)realloc(o->wt_cnt, sizeof(int32_t) * cap);
    o->consensus = (uint8_t *)realloc(o->consensus, cap);
    for (int i = o->rcap; i < cap; i++) {
        for (size_t c = 0; c < M; c++) o->wt[i * M + c] = -1;
        o->wt_cnt[i] = 0; o->consensus[i] = 0;
    }
    o->rcap = cap;
}

/* swirld.py:114-120 add_event (hg[h] = ev; tbd.add(h); height) */
int or_append(void *h, int n, const int32_t *p0, const int32_t *p1,
              const int32_t *creator, const double *t, const uint8_t *sig) {
    oracle *o = (oracle *)h;
    if (!o || n < 0) return OR_ERR_ARG;
    grow_events(o, o->n + n);
    for (int j = 0; j < n; j++) {
        int i = o->n + j;
        if (creator[j] < 0 || creator[j] >= o->M) return OR_ERR_ARG;
        if ((p0[j] < 0) != (p1[j] < 0) || p0[j] >= i || p1[j] >= i) return OR_ERR_ARG;
        o->p0[i] = p0[j]; o->p1[i] = p1[j]; o->creator[i] = creator[j];
        o->t[i] = t[j];
        memcpy(o->sig + (size_t)64 * i, sig + (size_t)64 * j, 64);
        o->tbd[i] = 1;                                         /* swirld.py:116 */
        if (p0[j] < 0) o->height[i] = 0;                       /* swirld.py:117-118 */
        else {
            int a = o->height[p0[j]], b = o->height[p1[j]];    /* swirld.py:120 */
            o->height[i] = (a > b ? a : b) + 1;
        }
        for (int c = 0; c < o->M; c++) o->can_see[(size_t)i * o->M + c] = -1;
    }
    o->n += n;
    return 0;
}

/* swirld.py:183-184 higher(a, b) with None == -1 */
static int higher(const oracle *o, int a, int b) {
    return a >= 0 && (b < 0 || o->height[a] >= o->height[b]);
}

/* self.witnesses[r][c] = h (dict assignment keeps first-insertion position) */
static void set_witness(oracle *o, int r, int c, int h) {
    grow_rounds(o, r);
    size_t M = (size_t)o->M;
    if (o->wt[r * M + c] < 0) o->wt_order[r * M + o->wt_cnt[r]++] = c;
    o->wt[r * M + c] = h;
    if (r > o->max_r) o->max_r = r;
}

/* the shared "count distinct paths" block, swirld.py:207-214 and 246-252:
 * hits[c_] += stake[c] for every (c,k) in can_see[h] with round[k]==r and every
 * (c_,k_) in can_see[k] with round[k_]==r. */
static void count_hits(oracle *o, int h, int r) {
    int M = o->M;
    const int32_t *row = o->can_see + (size_t)h * M;
    for (int c = 0; c < M; c++) o->hits[c] = 0;
    for (int c = 0; c < M; c++) {
        int k = row[c];
        if (k < 0 || o->round[k] != r) continue;
        const int32_t *rk = o->can_see + (size_t)k * M;
        for (int c_ = 0; c_ < M; c_++) {
            int k_ = rk[c_];
            if (k_ >= 0 && o->round[k_] == r) o->hits[c_] += o->stake[c];
        }
    }
}

/* swirld.py:187-222 */
int or_divide_rounds(void *hd, int first, int n) {
    oracle *o = (oracle *)hd;
    if (!o || first < 0 || n < 0 || first + n > o->n) return OR_ERR_ARG;
    int M = o->M;
    for (int h = first; h < first + n; h++) {
        int32_t *row = o->can_see + (size_t)h * M;
        int c = o->creator[h];
        if (o->p0[h] < 0) {                      /* swirld.py:195-198 root */
            o->round[h] = 0;
            set_witness(o, 0, c, h);
            for (int m = 0; m < M; m++) row[m] = -1;
            row[c] = h;
            continue;
        }
        int pa = o->p0[h], pb = o->p1[h];
        if (o->round[pa] < 0 || o->round[pb] < 0) return OR_ERR_KEY;
        int r = o->round[pa] > o->round[pb] ? o->round[pa] : o->round[pb];  /* :200 */
        const int32_t *ra = o->can_see + (size_t)pa * M;
        const int32_t *rb = o->can_see + (size_t)pb * M;
        for (int m = 0; m < M; m++) {             /* swirld.py:203-205, maxi 170-174 */
            int a = ra[m], b = rb[m];
            row[m] = (a < 0 && b < 0) ? -1 : (higher(o, a, b) ? a : b);
        }
        count_hits(o, h, r);                      /* swirld.py:208-214 */
        int cnt = 0;
        for (int m = 0; m < M; m++) if ((double)o->hits[m] > o->min_s) cnt++;
        o->round[h] = ((double)cnt > o->min_s) ? r + 1 : r;   /* swirld.py:216-219 */
        row[c] = h;                               /* swirld.py:220 */
        if (o->round[h] > o->round[pa])           /* swirld.py:221-222 */
            set_witness(o, o->round[h], c, h);
    }
    return 0;
}

static int cmp_i32(const void *a, const void *b) {
    int32_t x = *(const int32_t *)a, y = *(const int32_t *)b;
    return (x > y) - (x < y);
}

/* swirld.py:224-277.  Returns |new_c| (sorted into new_c_out), or <0. */
int or_decide_fame(void *hd, int32_t *new_c_out, int cap) {
    oracle *o = (oracle *)hd;
    if (!o) return OR_ERR_ARG;
    if (o->max_r < 0) return OR_ERR_ARG;       /* max() of empty dict raises */
    int M = o->M;
    int max_r = o->max_r;                       /* :225 */
    int max_c = 0;
    while (max_c < o->rcap && o->consensus[max_c]) max_c++;   /* :226-228 */
    uint8_t *done = (uint8_t *)calloc((size_t)max_r + 2, 1);  /* :243 */
    int32_t *s = (int32_t *)malloc(sizeof(int32_t) * M);

    for (int r_ = max_c + 1; r_ <= max_r; r_++) {             /* iter_voters :238-241 */
        for (int vi = 0; vi < o->wt_cnt[r_]; vi++) {
            int y = o->wt[(size_t)r_ * M + o->wt_order[(size_t)r_ * M + vi]];
            count_hits(o, y, r_ - 1);                         /* :245-251 */
            int ns = 0;                                       /* :252-253 */
            for (int c = 0; c < M; c++)
                if (o->hits[c] != 0 && (double)o->hits[c] > o->min_s) {
                    int w = o->wt[(size_t)(r_ - 1) * M + c];
                    if (w < 0) { free(done); free(s); return OR_ERR_KEY; }
                    s[ns++] = w;
                }
            for (int r = max_c; r < r_; r++) {                /* iter_undetermined :231-236 */
                if (o->consensus[r]) continue;
                for (int xi = 0; xi < o->wt_cnt[r]; xi++) {
                    int x = o->wt[(size_t)r * M + o->wt_order[(size_t)r * M + xi]];
                    if (o->famous[x] >= 0) continue;
                    if (r_ - r == 1) {                        /* :256-257 */
                        int in = 0;
                        for (int i = 0; i < ns; i++) if (s[i] == x) in = 1;
                        vm_put(&o->votes, (uint32_t)y, (uint32_t)x, in);
                    } else {
                        int64_t hv[2] = {0, 0};               /* majority :20-27 */
                        if (ns == 0) o->cov[OR_COV_MAJORITY_EMPTY]++;
                        for (int i = 0; i < ns; i++) {
                            int v = vm_get(&o->votes, (uint32_t)s[i], (uint32_t)x);
                            if (v < 0) { free(done); free(s); return OR_ERR_KEY; }
                            hv[v] += o->stake[o->creator[s[i]]];
                        }
                        int v; int64_t tt;
                        if (hv[0] > hv[1]) { v = 0; tt = hv[0]; } else { v = 1; tt = hv[1]; }
                        if ((r_ - r) % o->C != 0) {           /* :260 */
                            if ((double)tt > o->min_s) {      /* :261-263 */
                                o->famous[x] = (int8_t)v;
                                done[r] = 1;
                                o->cov[OR_COV_DECISIONS]++;
                                if (r_ - r > o->C) o->cov[OR_COV_DECIDE_AFTER_C]++;
                            } else
                                vm_put(&o->votes, (uint32_t)y, (uint32_t)x, v);
                        } else {
                            if ((double)tt > o->min_s) {      /* :267-268 */
                                vm_put(&o->votes, (uint32_t)y, (uint32_t)x, v);
                                o->cov[OR_COV_COIN_SUPER]++;
                            } else {                          /* :270-272 coin */
                                int coin = o->sig[(size_t)64 * y] / 128 ? 1 : 0;
                                vm_put(&o->votes, (uint32_t)y, (uint32_t)x, coin);
                                o->cov[OR_COV_COIN_VOTES]++;
                                o->cov[OR_COV_COIN_ONES] += coin;
                            }
                        }
                    }
                }
            }
        }
    }
    int nn = 0;
    for (int r = 0; r <= max_r; r++) {                        /* :274-276 */
        if (!done[r]) continue;
        int all = 1;
        for (int xi = 0; xi < o->wt_cnt[r]; xi++) {
            int x = o->wt[(size_t)r * M + o->wt_order[(size_t)r * M + xi]];
            if (o->famous[x] < 0) all = 0;
        }
        if (all) {
            if (nn < cap) new_c_out[nn] = r;
            nn++;
        }
    }
    int lim = nn < cap ? nn : cap;
    for (int i = 0; i < lim; i++) o->consensus[new_c_out[i]] = 1;
    free(done); free(s);
    return nn <= cap ? nn : OR_ERR_ARG;
}

/* sort keys of swirld.py:306: (ts[x], white ^ to_int(x)) */
typedef struct { double ts; uint8_t key[64]; int32_t x; } okey;
static int cmp_okey(const void *a, const void *b) {
    const okey *p = (const okey *)a, *q = (const okey *)b;
    if (p->ts < q->ts) return -1;
    if (p->ts > q->ts) return 1;
    int c = memcmp(p->key, q->key, 64);        /* big-endian 512-bit ints */
    if (c) return c;
    return (p->x > q->x) - (p->x < q->x);
}
static int cmp_dbl(const void *a, const void *b) {
    double x = *(const double *)a, y = *(const double *)b;
    return (x > y) - (x < y);
}

/* swirld.py:280-311 (the print at :310-311 is the caller's business) */
int or_find_order(void *hd, const int32_t *new_c, int n) {
    oracle *o = (oracle *)hd;
    if (!o || n < 0) return OR_ERR_ARG;
    int M = o->M;
    int32_t *rs = (int32_t *)malloc(sizeof(int32_t) * (n + 1));
    memcpy(rs, new_c, sizeof(int32_t) * n);
    qsort(rs, n, sizeof(int32_t), cmp_i32);                    /* sorted(new_c) :283 */
    int32_t *fw = (int32_t *)malloc(sizeof(int32_t) * M);
    int32_t *sw = (int32_t *)malloc(sizeof(int32_t) * M);
    double *times = (double *)malloc(sizeof(double) * M);
    int rc = 0;
    for (int ri = 0; ri < n && rc == 0; ri++) {
        int r = rs[ri];
        if (r < 0 || r > o->max_r) { rc = OR_ERR_KEY; break; }
        int nf = 0;
        uint8_t white[64];
        memset(white, 0, 64);
        for (int xi = 0; xi < o->wt_cnt[r]; xi++) {            /* :284 f_w */
            int w = o->wt[(size_t)r * M + o->wt_order[(size_t)r * M + xi]];
            if (o->famous[w] < 0) { rc = OR_ERR_KEY; break; }
            if (o->famous[w] == 1) {
                fw[nf++] = w;
                for (int b = 0; b < 64; b++) white[b] ^= o->sig[(size_t)64 * w + b];  /* :285 */
            }
        }
        if (rc) break;
        /* bfs over tbd from f_w & tbd, utils.py:24-34 and swirld.py:288-289 */
        int qh = 0, qt = 0;
        for (int i = 0; i < nf; i++)
            if (o->tbd[fw[i]] && !o->mark[fw[i]]) { o->mark[fw[i]] = 1; o->queue[qt++] = fw[i]; }
        okey *keys = NULL; int nk = 0, kcap = 0;
        while (qh < qt) {
            int x = o->queue[qh++];
            int c = o->creator[x];
            int ns = 0; int64_t st = 0;
            for (int i = 0; i < nf; i++) {                     /* :291-292 */
                int k = o->can_see[(size_t)fw[i] * M + c];
                if (k >= 0 && higher(o, k, x)) { sw[ns++] = fw[i]; st += o->stake[o->creator[fw[i]]]; }
            }
            int received = (double)st > (double)o->tot_stake / 2.0;   /* :293 */
            if (received) {
                o->tbd[x] = 0;                                 /* :294 */
                for (int i = 0; i < ns; i++) {                 /* :297-303 */
                    int a = sw[i];
                    for (;;) {
                        int k = o->can_see[(size_t)a * M + c];
                        if (k >= 0 && higher(o, k, x) && o->p0[a] >= 0) a = o->p0[a];
                        else break;
                    }
                    times[i] = o->t[a];
                }
                qsort(times, ns, sizeof(double), cmp_dbl);     /* :304 */
                if ((ns + 1) / 2 >= ns) { rc = OR_ERR_INDEX; o->cov[OR_COV_SINGLE_SEER]++; }  /* :305 IndexError */
                else {
                    o->cov[ns % 2 ? OR_COV_MEDIAN_ODD : OR_COV_MEDIAN_EVEN]++;
                    if (nk == kcap) { kcap = kcap ? kcap * 2 : 256; keys = (okey *)realloc(keys, sizeof(okey) * kcap); }
                    keys[nk].ts = .5 * (times[ns / 2] + times[(ns + 1) / 2]);
                    for (int b = 0; b < 64; b++) keys[nk].key[b] = white[b] ^ o->sig[(size_t)64 * x + b];
                    keys[nk].x = x;
                    nk++;
                }
            }
            /* successors: parents still in tbd (evaluated after x was handled) */
            if (o->p0[x] >= 0) {
                int pp[2] = { o->p0[x], o->p1[x] };
                for (int j = 0; j < 2; j++)
                    if (o->tbd[pp[j]] && !o->mark[pp[j]]) { o->mark[pp[j]] = 1; o->queue[qt++] = pp[j]; }
            }
            if (rc) break;
        }
        for (int i = 0; i < qt; i++) o->mark[o->queue[i]] = 0;
        if (rc == 0) {
            qsort(keys, nk, sizeof(okey), cmp_okey);           /* :306 */
            for (int i = 1; i < nk; i++)
                if (keys[i].ts == keys[i - 1].ts) o->cov[OR_COV_TIED]++;
            for (int i = 0; i < nk; i++) {                     /* :307-309 */
                o->idx[keys[i].x] = i + o->n_tx;
            }
            for (int i = 0; i < nk; i++) o->transactions[o->n_tx + i] = keys[i].x;
            o->n_tx += nk;
        }
        free(keys);
    }
    free(rs); free(fw); free(sw); free(times);
    return rc;
}

/* ---------------------------------------------------------------- getters */
int or_n_events(void *h) { return ((oracle *)h)->n; }
int or_max_round(void *h) { return ((oracle *)h)->max_r; }
int or_n_transactions(void *h) { return ((oracle *)h)->n_tx; }
/* copies the OR_NCOV branch counters to out; returns OR_NCOV */
int or_coverage(void *h, int64_t *out) { oracle *o = (oracle *)h; memcpy(out, o->cov, sizeof o->cov); return OR_NCOV; }

void or_get_round(void *h, int32_t *out) { oracle *o = (oracle *)h; memcpy(out, o->round, sizeof(int32_t) * o->n); }
void or_get_famous(void *h, int8_t *out) { oracle *o = (oracle *)h; memcpy(out, o->famous, o->n); }
void or_get_idx(void *h, int32_t *out) { oracle *o = (oracle *)h; memcpy(out, o->idx, sizeof(int32_t) * o->n); }
void or_get_height(void *h, int32_t *out) { oracle *o = (oracle *)h; memcpy(out, o->height, sizeof(int32_t) * o->n); }
void or_get_transactions(void *h, int32_t *out) { oracle *o = (oracle *)h; memcpy(out, o->transactions, sizeof(int32_t) * o->n_tx); }
void or_get_can_see(void *h, int first, int n, int32_t *out) {
    oracle *o = (oracle *)h;
    memcpy(out, o->can_see + (size_t)first * o->M, sizeof(int32_t) * (size_t)n * o->M);
}
/* witness flag per event: 1 iff it is currently a value of witnesses[r] for some r */
void or_get_witness(void *h, uint8_t *out) {
    oracle *o = (oracle *)h;
    memset(out, 0, o->n);
    for (int r = 0; r <= o->max_r; r++)
        for (int c = 0; c < o->M; c++) {
            int w = o->wt[(size_t)r * o->M + c];
            if (w >= 0) out[w] = 1;
        }
}
void or_get_witness_table(void *h, int32_t *out) {   /* (max_r+1) x M */
    oracle *o = (oracle *)h;
    if (o->max_r >= 0) memcpy(out, o->wt, sizeof(int32_t) * (size_t)(o->max_r + 1) * o->M);
}
int or_get_consensus(void *h, int32_t *out, int cap) {
    oracle *o = (oracle *)h; int n = 0;
    for (int r = 0; r < o->rcap; r++)
        if (o->consensus[r]) { if (n < cap) out[n] = r; n++; }
    return n;
}
