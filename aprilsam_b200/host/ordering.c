/* ordering.c -- fill-reducing elimination order of the pose graph (host C).
 *
 * The incremental solver's observable behaviour depends on the block elimination tree
 * (which nodes are "affected", whether back-substitution prunes, when a batch re-solve is
 * triggered -- SURVEY.md section 7 "Ordering leaks into incremental results"), so the drop-in
 * must produce the SAME permutation as the reference's heap_minimum_degree_ordering()
 * (aprilsam/aprilsam.c:999-1249).  This file is an independent implementation of that
 * procedure -- bucketed, lazily re-queued exact minimum degree with the newest pose and a
 * +-5 index window around its neighbours forced to the end -- using flat arrays instead of
 * the reference's hash table / heap-of-queues objects.  The tie-breaking rules that decide
 * the permutation are reproduced deliberately:
 *   - buckets are FIFO and are created in first-use order;
 *   - buckets are popped from a binary max-heap on (-key) as float, with the reference
 *     heap's sift rules (zmaxheap.c:134-159 insert: stop when parent >= v;
 *     :181-241 remove: move last to root, descend to the left child on ties);
 *   - a popped node whose degree grew past its bucket key is appended to the registered
 *     bucket of its new degree, or to a fresh UNREGISTERED bucket (aprilsam.c:1224-1234);
 *   - the window loop registers nodes 0..deg-1 (loop counter used as node id,
 *     aprilsam.c:1080-1094) without marking them.
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "asam_host.h"

/* FIFO bucket: a singly linked list of items drawn from one pool shared by all buckets (no per-bucket
 * allocation: a replay re-orders the graph at every batch escalation, thousands of buckets each time) */
typedef struct {
    int head, tail, n; /* indices into the item pool, -1 = none */
} bucket_t;

typedef struct {
    bucket_t *b;
    int nb, capb;
    int *reg; /* key -> bucket index, -1 if none */
    int nreg;
    float *hv; /* heap values */
    int *hb;   /* heap payload: bucket index */
    int hn, hcap;
    int *inode, *inext; /* item pool */
    int ni, icap;
} mdq_t;

static void heap_push(mdq_t *q, int bucket, float v)
{
    if (q->hn == q->hcap) {
        q->hcap = q->hcap ? 2 * q->hcap : 64;
        q->hv = realloc(q->hv, sizeof(float) * q->hcap);
        q->hb = realloc(q->hb, sizeof(int) * q->hcap);
    }
    int i = q->hn++;
    q->hv[i] = v;
    q->hb[i] = bucket;
    while (i > 0) {
        int p = (i - 1) / 2;
        if (q->hv[p] >= v)
            break;
        float tv = q->hv[p]; q->hv[p] = q->hv[i]; q->hv[i] = tv;
        int tb = q->hb[p]; q->hb[p] = q->hb[i]; q->hb[i] = tb;
        i = p;
    }
}

static int heap_pop(mdq_t *q, int *bucket, float *v)
{
    if (q->hn == 0)
        return 0;
    *bucket = q->hb[0];
    *v = q->hv[0];
    q->hn--;
    if (q->hn == 0)
        return 1;
    q->hv[0] = q->hv[q->hn];
    q->hb[0] = q->hb[q->hn];
    int p = 0;
    float ps = q->hv[0];
    for (;;) {
        int l = 2 * p + 1, r = l + 1;
        float ls = l < q->hn ? q->hv[l] : -INFINITY;
        float rs = r < q->hn ? q->hv[r] : -INFINITY;
        if (ps >= ls && ps >= rs)
            break;
        int c = (ls >= rs) ? l : r;
        float tv = q->hv[p]; q->hv[p] = q->hv[c]; q->hv[c] = tv;
        int tb = q->hb[p]; q->hb[p] = q->hb[c]; q->hb[c] = tb;
        p = c;
    }
    return 1;
}

static int bucket_new(mdq_t *q)
{
    if (q->nb == q->capb) {
        q->capb = q->capb ? 2 * q->capb : 64;
        q->b = realloc(q->b, sizeof(bucket_t) * q->capb);
    }
    bucket_t *b = &q->b[q->nb];
    b->head = b->tail = -1;
    b->n = 0;
    return q->nb++;
}

static void bucket_push(mdq_t *q, int bi, int node)
{
    if (q->ni == q->icap) {
        q->icap = q->icap ? 2 * q->icap : 1024;
        q->inode = realloc(q->inode, sizeof(int) * (size_t) q->icap);
        q->inext = realloc(q->inext, sizeof(int) * (size_t) q->icap);
    }
    const int it = q->ni++;
    q->inode[it] = node;
    q->inext[it] = -1;
    bucket_t *b = &q->b[bi];
    if (b->tail >= 0)
        q->inext[b->tail] = it;
    else
        b->head = it;
    b->tail = it;
    b->n++;
}

/* pop the oldest item of a non-empty bucket */
static inline int bucket_pop(mdq_t *q, int bi)
{
    bucket_t *b = &q->b[bi];
    const int it = b->head;
    b->head = q->inext[it];
    if (b->head < 0)
        b->tail = -1;
    b->n--;
    return q->inode[it];
}

/* enqueue into the registered bucket of `key`, creating + registering it on first use */
static void enqueue_registered(mdq_t *q, unsigned key, int node)
{
    if ((int) key >= q->nreg) {
        int nn = q->nreg;
        while (nn <= (int) key)
            nn *= 2;
        q->reg = realloc(q->reg, sizeof(int) * nn);
        for (int i = q->nreg; i < nn; i++)
            q->reg[i] = -1;
        q->nreg = nn;
    }
    int bi = q->reg[key];
    if (bi < 0) {
        bi = bucket_new(q);
        q->reg[key] = bi;
        bucket_push(q, bi, node);
        heap_push(q, bi, (float) (-1.0 * key));
    } else {
        bucket_push(q, bi, node);
    }
}

/* First implementation: explicit elimination graph (every elimination turns the neighbours into a
 * clique).  O(sum d^2); kept as the cross-check of the quotient-graph version below (tests). */
int *asam_ref_ordering_explicit(int N, const int *adj_ptr, const int *adj)
{
    int *order = calloc(N > 0 ? N : 1, sizeof(int));
    if (N <= 0)
        return order;

    /* mutable neighbour lists of the elimination graph */
    int **nbr = malloc(sizeof(int *) * N);
    int *deg = malloc(sizeof(int) * N);
    int *cap = malloc(sizeof(int) * N);
    for (int i = 0; i < N; i++) {
        int d = adj_ptr[i + 1] - adj_ptr[i];
        cap[i] = 2 * d + 8;
        nbr[i] = malloc(sizeof(int) * cap[i]);
        memcpy(nbr[i], adj + adj_ptr[i], sizeof(int) * d);
        deg[i] = d;
    }

    mdq_t q;
    memset(&q, 0, sizeof(q));
    q.nreg = 3 * N + 16;
    q.reg = malloc(sizeof(int) * q.nreg);
    for (int i = 0; i < q.nreg; i++)
        q.reg[i] = -1;

    char *pinned = calloc(N, 1);
    {
        /* newest pose last; a window of +-5 ids around each of its neighbours late */
        int last = N - 1;
        enqueue_registered(&q, (unsigned) (deg[last] + 2 * last), last);
        pinned[last] = 1;
        for (int i = 0; i < deg[last]; i++) {
            int c = nbr[last][i];
            for (int idx = c - 5; idx < c + 5; idx++) {
                if (idx < 0 || idx > N - 1 || pinned[idx])
                    continue;
                enqueue_registered(&q, (unsigned) (deg[idx] + last), idx);
                pinned[idx] = 1;
                for (int j = 0; j < deg[idx]; j++) { /* j is used as a node id (reference quirk) */
                    if (pinned[j])
                        continue;
                    enqueue_registered(&q, (unsigned) (deg[j] + last), j);
                }
            }
        }
    }
    for (int r = 0; r < N - 1; r++)
        if (!pinned[r])
            enqueue_registered(&q, (unsigned) deg[r], r);
    free(pinned);

    char *gone = calloc(N, 1);
    int *stamp = calloc(N, sizeof(int));
    int token = 0, k = 0;
    int bi;
    float v;
    while (heap_pop(&q, &bi, &v)) {
        while (q.b[bi].n > 0) {
            int u = bucket_pop(&q, bi);
            if (gone[u])
                continue;
            if ((float) deg[u] <= -v) {
                order[k++] = u;
                gone[u] = 1;
                /* eliminate u: its neighbours become a clique */
                for (int ai = 0; ai < deg[u]; ai++) {
                    int a = nbr[u][ai];
                    token++;
                    int *na = nbr[a];
                    for (int i = 0; i < deg[a]; i++) {
                        if (na[i] == u) {
                            na[i] = na[deg[a] - 1];
                            deg[a]--;
                            i--;
                            continue;
                        }
                        stamp[na[i]] = token;
                    }
                    stamp[u] = token;
                    stamp[a] = token;
                    for (int bj = 0; bj < deg[u]; bj++) {
                        int w = nbr[u][bj];
                        if (stamp[w] == token)
                            continue;
                        if (deg[a] + 1 >= cap[a]) {
                            cap[a] *= 2;
                            nbr[a] = realloc(nbr[a], sizeof(int) * cap[a]);
                        }
                        nbr[a][deg[a]++] = w;
                    }
                }
            } else {
                unsigned key = (unsigned) deg[u];
                int rb = ((int) key < q.nreg) ? q.reg[key] : -1;
                if (rb >= 0) {
                    bucket_push(&q, rb, u);
                } else {
                    int nb = bucket_new(&q); /* not registered: later re-queues make more */
                    bucket_push(&q, nb, u);
                    heap_push(&q, nb, (float) (-1.0 * key));
                }
            }
        }
    }
    /* any node never reached (cannot happen for a valid graph) goes last, in id order */
    if (k < N) {
        for (int i = 0; i < N; i++)
            if (!gone[i])
                order[k++] = i;
    }

    for (int i = 0; i < N; i++)
        free(nbr[i]);
    free(q.inode);
    free(q.inext);
    free(q.b);
    free(q.reg);
    free(q.hv);
    free(q.hb);
    free(nbr);
    free(deg);
    free(cap);
    free(gone);
    free(stamp);
    return order;
}

/* ---- quotient-graph version ------------------------------------------------------------------
 * Same queue discipline (the code above and the pop / re-queue logic below are what fixes the
 * permutation), but the elimination graph is kept implicitly: an eliminated pose u becomes an
 * ELEMENT whose member list L_u is its set of neighbours at elimination time; a live pose v keeps
 * the original neighbours not yet covered by an element (A_v) and the elements it belongs to (E_v);
 * elements adjacent to u are absorbed into L_u.  The exact degree |A_v u U_{e in E_v} L_e| is
 * evaluated only when v is popped (the queue is lazy anyway), by marking.  A live element never
 * holds an eliminated pose (eliminating a member absorbs the element), nor does any A_v.
 * Work is O(sum |L|) per elimination / pop instead of O(d^2). */
/* storage: A_v and E_v share the slot of deg0(v) ints that held v's original neighbour list (A_v
 * from the front, E_v from the back: |A_v| + |E_v| <= deg0(v) always, because a pose enters an
 * element only by losing a neighbour entry or an absorbed element); the member lists L_u come from a
 * bump pool (sum |L_u| = number of block non-zeros of the factor).  No per-pose malloc. */
int *asam_ref_ordering(int N, const int *adj_ptr, const int *adj)
{
    int *order = calloc(N > 0 ? N : 1, sizeof(int));
    if (N <= 0)
        return order;

    const int S2 = adj_ptr[N];
    int *slot = malloc(sizeof(int) * (size_t) (S2 + 1));
    memcpy(slot, adj, sizeof(int) * (size_t) S2);
    int *an = malloc(sizeof(int) * (size_t) N);  /* |A_v| */
    int *en = calloc((size_t) N, sizeof(int));   /* |E_v| */
    int *deg0 = malloc(sizeof(int) * (size_t) N);
    for (int i = 0; i < N; i++)
        an[i] = deg0[i] = adj_ptr[i + 1] - adj_ptr[i];
#define A_OF(v) (slot + adj_ptr[v])
#define E_OF(v) (slot + adj_ptr[(v) + 1] - en[v]) /* en[v] entries ending at the slot's end */
    int64_t lcap = 4 * (int64_t) S2 + 1024, ln = 0;
    int *lpool = malloc(sizeof(int) * (size_t) lcap);
    int64_t *loff = malloc(sizeof(int64_t) * (size_t) N); /* element u: lpool[loff[u] .. +llen[u]) */
    int *llen = calloc((size_t) N, sizeof(int));
    char *dead = calloc((size_t) N, 1);

    mdq_t q;
    memset(&q, 0, sizeof(q));
    q.nreg = 3 * N + 16;
    q.reg = malloc(sizeof(int) * q.nreg);
    for (int i = 0; i < q.nreg; i++)
        q.reg[i] = -1;

    char *pinned = calloc(N, 1);
    {
        /* newest pose last; a window of +-5 ids around each of its neighbours late */
        int last = N - 1;
        enqueue_registered(&q, (unsigned) (deg0[last] + 2 * last), last);
        pinned[last] = 1;
        for (int i = 0; i < deg0[last]; i++) {
            int c = A_OF(last)[i];
            for (int idx = c - 5; idx < c + 5; idx++) {
                if (idx < 0 || idx > N - 1 || pinned[idx])
                    continue;
                enqueue_registered(&q, (unsigned) (deg0[idx] + last), idx);
                pinned[idx] = 1;
                for (int j = 0; j < deg0[idx]; j++) { /* j is used as a node id (reference quirk) */
                    if (pinned[j])
                        continue;
                    enqueue_registered(&q, (unsigned) (deg0[j] + last), j);
                }
            }
        }
    }
    for (int r = 0; r < N - 1; r++)
        if (!pinned[r])
            enqueue_registered(&q, (unsigned) deg0[r], r);
    free(pinned);

    char *gone = calloc(N, 1);
    int *stamp = calloc(N, sizeof(int));
    int token = 0, k = 0;
    int bi;
    float v;
    while (heap_pop(&q, &bi, &v)) {
        while (q.b[bi].n > 0) {
            int u = bucket_pop(&q, bi);
            if (gone[u])
                continue;
            /* exact degree of u now; its element list is compacted on the way */
            int du = 0;
            token++;
            stamp[u] = token;
            const int *Au = A_OF(u);
            for (int i = 0; i < an[u]; i++) {
                int w = Au[i];
                if (stamp[w] != token) {
                    stamp[w] = token;
                    du++;
                }
            }
            {
                /* E_u sits at the END of the slot: compact towards the end, keeping the order */
                int *Eu = E_OF(u), ne = 0;
                for (int i = en[u] - 1; i >= 0; i--) {
                    int e = Eu[i];
                    if (dead[e])
                        continue;
                    Eu[en[u] - 1 - ne] = e;
                    ne++;
                }
                en[u] = ne;
                Eu = E_OF(u);
                for (int i = 0; i < ne; i++) {
                    int e = Eu[i];
                    const int *Le = lpool + loff[e];
                    for (int j = 0; j < llen[e]; j++) {
                        int w = Le[j];
                        if (stamp[w] != token) {
                            stamp[w] = token;
                            du++;
                        }
                    }
                }
            }
            if ((float) du <= -v) {
                order[k++] = u;
                gone[u] = 1;
                /* eliminate u: L_u = everything marked above (stamp == token) except u itself */
                stamp[u] = -token; /* u itself is a member of every element in E_u: not of L_u */
                if (ln + du > lcap) {
                    while (ln + du > lcap)
                        lcap *= 2;
                    lpool = realloc(lpool, sizeof(int) * (size_t) lcap);
                }
                int *Lu = lpool + ln;
                int nl = 0;
                for (int i = 0; i < an[u]; i++) {
                    int w = Au[i];
                    if (stamp[w] == token) { /* first visit collects, stamp flipped to avoid duplicates */
                        stamp[w] = -token;
                        Lu[nl++] = w;
                    }
                }
                const int *Eu = E_OF(u);
                for (int i = 0; i < en[u]; i++) {
                    int e = Eu[i];
                    const int *Le = lpool + loff[e];
                    for (int j = 0; j < llen[e]; j++) {
                        int w = Le[j];
                        if (stamp[w] == token) {
                            stamp[w] = -token;
                            Lu[nl++] = w;
                        }
                    }
                    dead[e] = 1; /* absorbed */
                }
                loff[u] = ln;
                llen[u] = nl;
                ln += nl;
                an[u] = en[u] = 0;
                /* members: drop neighbours now covered by the new element, swap absorbed elements for it */
                for (int i = 0; i < nl; i++) {
                    int m = Lu[i], na = 0;
                    int *Am = A_OF(m);
                    for (int j = 0; j < an[m]; j++)
                        if (stamp[Am[j]] != -token)
                            Am[na++] = Am[j];
                    an[m] = na;
                    int *Em = E_OF(m), ne = 0;
                    for (int j = en[m] - 1; j >= 0; j--) {
                        int e = Em[j];
                        if (dead[e])
                            continue;
                        Em[en[m] - 1 - ne] = e;
                        ne++;
                    }
                    en[m] = ne + 1;
                    *E_OF(m) = u; /* one position further down: room is guaranteed (see above) */
                }
            } else {
                unsigned key = (unsigned) du;
                int rb = ((int) key < q.nreg) ? q.reg[key] : -1;
                if (rb >= 0) {
                    bucket_push(&q, rb, u);
                } else {
                    int nb = bucket_new(&q); /* not registered: later re-queues make more */
                    bucket_push(&q, nb, u);
                    heap_push(&q, nb, (float) (-1.0 * key));
                }
            }
        }
    }
    /* any node never reached (cannot happen for a valid graph) goes last, in id order */
    if (k < N) {
        for (int i = 0; i < N; i++)
            if (!gone[i])
                order[k++] = i;
    }
#undef A_OF
#undef E_OF
    free(q.inode);
    free(q.inext);
    free(q.b);
    free(q.reg);
    free(q.hv);
    free(q.hb);
    free(slot);
    free(an);
    free(en);
    free(deg0);
    free(lpool);
    free(loff);
    free(llen);
    free(dead);
    free(gone);
    free(stamp);
    return order;
}
