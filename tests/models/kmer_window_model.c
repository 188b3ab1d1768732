/* tests/models/kmer_window_model.c -- TEST INFRASTRUCTURE: a scalar CPU model of the device algorithm of
 * k_kmer_window (filtlong_b200/csrc/fl_score.cu), which computes the k-mer-mode window quality of
 * read.cpp:216-236 bit for bit WITHOUT walking a row base by base.
 *
 * The reference's recurrence on qualities in {0, 1}:   w -= out ? rq : 0;  w += in ? rq : 0;  best = min(best, w)
 * with rq = fl(1 / ws), started from w0 = fl(c0 / ws). Let c be the window's hit count (an integer prefix
 * sum of the mask: parallel). Facts used (IEEE-754 round to nearest even; "grid" of a binade = its ulp):
 *
 *  (1) inside one binade adding / subtracting rq moves w by exactly R = rq rounded to the binade's grid: the two
 *      are inverse. Also in a "tie binade" (rq = (n + 1/2) grid units exactly): round-half-even makes every result
 *      of an operation there EVEN, and from an even value the step is the even one of n, n + 1;
 *  (2) subtracting rq across a binade edge (the lower grid is finer, w is on it) and adding it back returns
 *      to the same value (the two roundings compose to the identity whatever the parity: see DESIGN.md);
 *  (3) so, starting from an ANCHOR (w_a, c_a), every value the chain takes at a level c that is reached by
 *      moves BELOW the highest level visited since the anchor is one fixed function F(c): the
 *      value obtained by walking from the anchor down (or up, inside the anchor's binade) to c. The chain's
 *      minimum over such a stretch ("epoch") is F(min c) -- one count reduction and one short walk;
 *  (4) what is NOT reversible: an addition that takes the chain to a level it has not visited since the anchor
 *      AND sits next to a binade edge -- it either carries w into the coarser grid above (which forgets the
 *      low bit) or leaves the binade's lowest level (the subtraction that would undo it falls through the
 *      floor onto the finer grid); a new epoch starts from the value it produced. And an ODD value inside a tie
 *      binade (the first one after entering from the finer grid below, or w0 itself): nothing is reversible
 *      until an operation has made it even. Only THAT step is done with true double operations (the chain's
 *      value before it is F, the value after it is the new anchor); such steps are rare (a handful of record
 *      levels per row).
 *
 * The model processes a row in words of 32 steps exactly like one lane of the kernel does (word statistics
 * from a nibble look-up table, a predicate that flags the word; a flagged word is searched for its
 * irreversible step(s), which the kernel does with one lane per step), so that the CUDA code is a transcription
 * of this file.
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

/* one edge for every binade from rq's own up to 2^1: at most 33 for a window size below 2^31 (rq >= 2^-31). Dropping
 * one would let the chain cross that edge as if it were inside a binade (a window quality one ulp off at ws >= 2^15). */
#define KW_MAX_EDGES 34

typedef struct {
    double rq;
    int e_rq;             /* rq in [2^e_rq, 2^(e_rq+1)) */
    uint64_t mant_rq;     /* 53-bit significand of rq */
    int n_edges;          /* count intervals around the binade edges 2^e / rq (two levels of margin) */
    int elo[KW_MAX_EDGES], ehi[KW_MAX_EDGES];
} chain_consts;

typedef struct {
    double w;             /* anchor value */
    int c;                /* anchor count */
    int lattice;          /* anchor's binade has a usable grid (above rq's own binade, not a tie binade) */
    int64_t wb, rint, lo, hi;
    int c_edge;           /* highest level reachable from the anchor without leaving its binade upwards (conservative) */
    int unsafe;           /* odd value inside a tie binade: nothing is reversible until an operation made it even */
} anchor_t;

static inline int64_t d2b(double x) { int64_t b; memcpy(&b, &x, 8); return b; }
static inline double b2d(int64_t b) { double x; memcpy(&x, &b, 8); return x; }

void kw_consts(chain_consts *k, int ws) {
    k->rq = 1.0 / (double)ws;
    const int64_t b = d2b(k->rq);
    k->e_rq = (int)((b >> 52) & 0x7FF) - 1023;
    k->mant_rq = ((uint64_t)b & ((1ull << 52) - 1ull)) | (1ull << 52);
    k->n_edges = 0;
    for (int e = k->e_rq; e <= 1 && k->n_edges < KW_MAX_EDGES; ++e) {           /* edges 2^e for every binade a count 0..ws can reach */
        const double x = ldexp(1.0, e) * (double)ws;
        if (x > (double)ws + 3.0) break;
        k->elo[k->n_edges] = (int)floor(x) - 2;
        k->ehi[k->n_edges] = (int)ceil(x) + 2;
        k->n_edges++;
    }
}

static inline int touches_edge(const chain_consts *k, int lo, int hi) {
    for (int i = 0; i < k->n_edges; ++i)
        if (lo <= k->ehi[i] && hi >= k->elo[i]) return 1;
    return 0;
}

/* grid parameters of the binade of w; returns 0 if it has none (rq's own binade and below: arithmetic there is exact) */
static int binade_of(const chain_consts *k, double w, int64_t *wb, int64_t *rint, int64_t *lo, int64_t *hi) {
    if (!(w > 0.0)) return 0;
    const int64_t b = d2b(w);
    const int e = (int)((b >> 52) & 0x7FF) - 1023;
    const int s = e - k->e_rq;
    if (s < 1 || s > 52) return 0;
    const uint64_t half = 1ull << (s - 1);
    int64_t r = (int64_t)((k->mant_rq + half) >> s);
    if ((k->mant_rq & ((1ull << s) - 1ull)) == half) {
        /* tie binade: rq = (n + 1/2) grid units. Round-half-even makes every result of an operation inside the binade
         * EVEN, and from an even value adding / subtracting rq moves by the even one of n, n + 1: a lattice again.
         * An odd value (only the first one after entering from the finer grid below, or the initial w0) has none. */
        if (b & 1) return 0;
        const int64_t n = (int64_t)(k->mant_rq >> s);
        r = (n & 1) ? n + 1 : n;
    }
    *wb = b;
    *rint = r;
    *lo = (int64_t)(e + 1023) << 52;
    *hi = *lo + (1ll << 52);
    return 1;
}

static void set_anchor(anchor_t *a, const chain_consts *k, double w, int c) {
    a->w = w;
    a->c = c;
    a->lattice = binade_of(k, w, &a->wb, &a->rint, &a->lo, &a->hi);
    a->unsafe = 0;
    if (!a->lattice && w > 0.0) {
        const int64_t b = d2b(w);
        const int s = (int)((b >> 52) & 0x7FF) - 1023 - k->e_rq;
        if (s >= 1 && s <= 52 && (k->mant_rq & ((1ull << s) - 1ull)) == (1ull << (s - 1))) a->unsafe = 1;
    }
    a->c_edge = c;                                                   /* no usable grid: any level above the anchor ends the epoch */
    if (a->lattice) a->c_edge = c + (int)((a->hi - 2 - a->wb) / a->rint);
}

/* F(c) for c <= a->c_edge: the chain's value at level c inside the anchor's epoch */
static double eval_F(const anchor_t *a, const chain_consts *k, int c, long long *n_true_ops) {
    if (c >= a->c) return a->lattice ? b2d(a->wb + a->rint * (int64_t)(c - a->c)) : a->w;   /* (c > a->c only with a grid) */
    double w = a->w;
    int cur = a->c;
    while (cur > c) {                                                /* walk down: grid jumps inside a binade, true subtractions at its floor */
        int64_t wb, rint, lo, hi;
        if (binade_of(k, w, &wb, &rint, &lo, &hi)) {
            int64_t room = (wb - (lo + 1)) / rint;                   /* levels that can be descended while staying >= lo + 1 */
            if (room > (int64_t)(cur - c)) room = cur - c;
            if (room > 0) {
                w = b2d(wb - rint * room);
                cur -= (int)room;
                continue;
            }
        }
        w = w - k->rq;                                               /* read.cpp:229 */
        ++*n_true_ops;
        --cur;
    }
    return w;
}

/* nibble table: for 4 steps with pure-plus bits p and pure-minus bits m (p & m == 0): packed
 * (delta + 4) | (min_after + 4) << 4 | (max_after + 4) << 8, min / max over the after-step partial sums */
static uint16_t g_lut[256];
static int g_lut_ready = 0;
static void build_lut(void) {
    for (int p = 0; p < 16; ++p)
        for (int m = 0; m < 16; ++m) {
            int d = 0, mn = 99, mx = -99;
            for (int t = 0; t < 4; ++t) {
                d += ((p >> t) & 1) - ((m >> t) & 1);
                if (d < mn) mn = d;
                if (d > mx) mx = d;
            }
            g_lut[p | (m << 4)] = (uint16_t)((d + 4) | ((mn + 4) << 4) | ((mx + 4) << 8));
        }
    g_lut_ready = 1;
}

static void word_stats(uint32_t pin, uint32_t pout, int *delta, int *mn, int *mx) {
    int d = 0, lo = 99, hi = -99;
    for (int k = 0; k < 8; ++k) {
        const unsigned e = g_lut[((pin >> (4 * k)) & 15u) | (((pout >> (4 * k)) & 15u) << 4)];
        const int dd = (int)(e & 15u) - 4, m0 = (int)((e >> 4) & 15u) - 4, m1 = (int)((e >> 8) & 15u) - 4;
        if (d + m0 < lo) lo = d + m0;
        if (d + m1 > hi) hi = d + m1;
        d += dd;
    }
    *delta = d; *mn = lo; *mx = hi;
}

/* window quality (already x 100) of the row [S, E) of a hit mask (bit i of mask[i >> 5] = base i covered) */
double kmer_window_model(const uint32_t *mask, int S, int E, int ws, long long *n_true_ops_out, long long *n_slow_words_out) {
    if (!g_lut_ready) build_lut();
    const int len = E - S;
    long long n_true = 0, n_slow = 0;
#define BIT(i) ((mask[(i) >> 5] >> ((i) & 31)) & 1u)
    if (len <= ws) {                                                   /* read.cpp:217-218 */
        long long hits = 0;
        for (int i = S; i < E; ++i) hits += BIT(i);
        if (n_true_ops_out) *n_true_ops_out = 0;
        if (n_slow_words_out) *n_slow_words_out = 0;
        return 100.0 * (double)hits / (double)len;
    }
    chain_consts k;
    kw_consts(&k, ws);
    int c = 0;
    for (int i = S; i < S + ws; ++i) c += BIT(i);
    double best = (double)c / (double)ws;                              /* read.cpp:220-223 */
    anchor_t a;
    set_anchor(&a, &k, best, c);
    int cmin = c;                                                      /* lowest after-step count of the current epoch */
    int trec = c;                                                      /* highest level visited since the anchor */
    const int T = len - ws;                                            /* steps: in = base S+ws+t, out = base S+t */
    for (int t0 = 0; t0 < T; t0 += 32) {
        uint32_t in = 0, out = 0;
        const int nv = T - t0 < 32 ? T - t0 : 32;
        for (int j = 0; j < nv; ++j) {
            in |= BIT(S + ws + t0 + j) << j;
            out |= BIT(S + t0 + j) << j;
        }
        const uint32_t pin = in & ~out, pout = out & ~in, both = in & out;
        int delta, mn, mx;
        word_stats(pin, pout, &delta, &mn, &mx);
        const int mn0 = mn < 0 ? mn : 0, mx0 = mx > 0 ? mx : 0;
        /* levels the word visits, including the dip of a step that subtracts and adds in the same step */
        const int lo_level = c + mn0 - (both ? 1 : 0), hi_level = c + mx0;
        const int flagged = (a.unsafe && (in | out)) ||
                            (hi_level > trec && (hi_level > a.c_edge || touches_edge(&k, trec, hi_level)));
        if (!flagged) {
            if (c + mn < cmin) cmin = c + mn;
            if (hi_level > trec) trec = hi_level;
            c += delta;
            continue;
        }
        ++n_slow;
        /* Only the step that does something irreversible is done with the reference's own operations: the first step that
         * reaches a level whose first visit ends the epoch (or, from an odd value in a tie binade, the first step that does
         * anything). Everything before it in the word is still inside the epoch (F), everything after it belongs to the
         * epoch of the new anchor -- which may end in this very word again. */
        {
            int p = 0, level = c;                                      /* next step to look at, level before it */
            for (;;) {
                int ts = -1, lv = level, seg_min = 0x7FFFFFFF, seg_max = -0x7FFFFFFF, rec = trec;
                for (int t = p; t < 32; ++t) {
                    const int o = (int)((out >> t) & 1u), i = (int)((in >> t) & 1u);
                    const int after = lv - o + i;
                    int stop;
                    if (a.unsafe) stop = o | i;
                    else stop = after > rec && (after > a.c_edge || touches_edge(&k, after, after));
                    if (stop) { ts = t; break; }
                    lv = after;
                    if (lv < seg_min) seg_min = lv;
                    if (lv > seg_max) seg_max = lv;
                    if (lv > rec) rec = lv;
                }
                if (seg_min < cmin) cmin = seg_min;
                if (seg_max > trec) trec = seg_max;
                if (ts < 0) { level = lv; break; }
                {
                    const double f = eval_F(&a, &k, cmin, &n_true);        /* close the epoch */
                    if (f < best) best = f;
                }
                double w = eval_F(&a, &k, lv, &n_true);                   /* the chain's value before step ts */
                if ((out >> ts) & 1u) { w -= k.rq; --lv; ++n_true; }      /* read.cpp:229 */
                if ((in >> ts) & 1u) { w += k.rq; ++lv; ++n_true; }       /* read.cpp:230 */
                if (w < best) best = w;                                   /* read.cpp:231-232 */
                set_anchor(&a, &k, w, lv);
                cmin = lv;
                trec = lv;
                level = lv;
                p = ts + 1;
            }
            c = level;
        }
    }
    {
        const double f = eval_F(&a, &k, cmin, &n_true);
        if (f < best) best = f;
    }
#undef BIT
    if (best < 0.5 / (double)ws) best = 0.0;                           /* read.cpp:233-234 */
    if (n_true_ops_out) *n_true_ops_out = n_true;
    if (n_slow_words_out) *n_slow_words_out = n_slow;
    return 100.0 * best;
}

/* the reference recurrence itself (read.cpp:216-236 on {0, 1} qualities), for the comparison */
double kmer_window_reference(const uint32_t *mask, int S, int E, int ws) {
#define BIT(i) ((mask[(i) >> 5] >> ((i) & 31)) & 1u)
    const int len = E - S;
    if (len <= ws) {
        long long hits = 0;
        for (int i = S; i < E; ++i) hits += BIT(i);
        return 100.0 * (double)hits / (double)len;
    }
    double sum = 0.0;
    for (int i = S; i < S + ws; ++i) sum += BIT(i) ? 1.0 : 0.0;
    double w = sum / (double)ws, best = w;
    for (int t = 0; t < len - ws; ++t) {
        const double qo = BIT(S + t) ? 1.0 : 0.0, qi = BIT(S + ws + t) ? 1.0 : 0.0;
        w -= qo / (double)ws;
        w += qi / (double)ws;
        if (w < best) best = w;
    }
    if (best < 0.5 / (double)ws) best = 0.0;
    return 100.0 * best;
#undef BIT
}
