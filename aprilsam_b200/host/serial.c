/* serial.c -- attributes, the stype registry and the ".graph" file format (host C, no GPU).
 *
 * SURVEY.md section 8(f) items 1-2: with these the reference's example programs link against this
 * library unchanged and data/M3500.graph loads natively.  Own implementation of the format
 * described by the reference (file:line cited per function); the attribute table is a small
 * insertion-ordered array instead of the reference's zhash.
 */
#include <inttypes.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "asam_host.h"
#include "common/stype.h"

/* ---- big-endian primitives (common/encode_bytes.h) ---------------------------------------- */
ASAM_API void encode_u8(uint8_t *out, uint32_t *pos, uint8_t v)
{
    if (out)
        out[*pos] = v;
    *pos += 1;
}

ASAM_API void encode_u32(uint8_t *out, uint32_t *pos, uint32_t v)
{
    if (out)
        for (int i = 0; i < 4; i++)
            out[*pos + i] = (uint8_t) (v >> (24 - 8 * i));
    *pos += 4;
}

ASAM_API void encode_u64(uint8_t *out, uint32_t *pos, uint64_t v)
{
    if (out)
        for (int i = 0; i < 8; i++)
            out[*pos + i] = (uint8_t) (v >> (56 - 8 * i));
    *pos += 8;
}

ASAM_API void encode_f64(uint8_t *out, uint32_t *pos, double v)
{
    uint64_t u;
    memcpy(&u, &v, 8);
    encode_u64(out, pos, u);
}

ASAM_API void encode_string_u32(uint8_t *out, uint32_t *pos, const char *s)
{
    uint32_t len = (uint32_t) strlen(s);
    encode_u32(out, pos, len);
    if (out)
        memcpy(out + *pos, s, len);
    *pos += len;
}

/* reads past the end yield 0, like the reference (encode_bytes.h:35-37 etc.) */
ASAM_API uint8_t decode_u8(const uint8_t *in, uint32_t *pos, uint32_t len)
{
    if (*pos + 1 > len)
        return 0;
    return in[(*pos)++];
}

ASAM_API uint32_t decode_u32(const uint8_t *in, uint32_t *pos, uint32_t len)
{
    if (*pos + 4 > len)
        return 0;
    uint32_t v = 0;
    for (int i = 0; i < 4; i++)
        v = (v << 8) | in[(*pos)++];
    return v;
}

ASAM_API uint64_t decode_u64(const uint8_t *in, uint32_t *pos, uint32_t len)
{
    if (*pos + 8 > len)
        return 0;
    uint64_t v = 0;
    for (int i = 0; i < 8; i++)
        v = (v << 8) | in[(*pos)++];
    return v;
}

ASAM_API double decode_f64(const uint8_t *in, uint32_t *pos, uint32_t len)
{
    uint64_t u = decode_u64(in, pos, len);
    double v;
    memcpy(&v, &u, 8);
    return v;
}

ASAM_API char *decode_string_u32(const uint8_t *in, uint32_t *pos, uint32_t len)
{
    uint32_t n = decode_u32(in, pos, len);
    if (*pos + n > len)
        return NULL;
    char *s = malloc((size_t) n + 1);
    memcpy(s, in + *pos, n);
    s[n] = 0;
    *pos += n;
    return s;
}

/* ---- registry (common/stype.c:49-73) ---------------------------------------------------------- */
static const stype_t **g_types;
static int g_ntypes, g_types_cap;

ASAM_API void stype_register(const stype_t *st)
{
    for (int i = 0; i < g_ntypes; i++)
        if (!strcmp(g_types[i]->name, st->name)) {
            g_types[i] = st;
            return;
        }
    if (g_ntypes == g_types_cap) {
        g_types_cap = g_types_cap ? 2 * g_types_cap : 16;
        g_types = realloc(g_types, sizeof(*g_types) * (size_t) g_types_cap);
    }
    g_types[g_ntypes++] = st;
}

ASAM_API stype_t *stype_get(char *name)
{
    for (int i = 0; name && i < g_ntypes; i++)
        if (!strcmp(g_types[i]->name, name))
            return (stype_t *) g_types[i];
    return NULL;
}

/* ---- framing (common/stype.c:75-169) ----------------------------------------------------------- */
ASAM_API void stype_encode_object(uint8_t *data, uint32_t *datapos, const stype_t *st, const void *obj)
{
    static uint64_t next_magic = 0x7b287f8a1579a0edULL; /* same cookie sequence as the reference */
    if (obj && !st)
        asam_fatal("stype_encode_object: object without a type");
    uint64_t magic = next_magic++;
    encode_u64(data, datapos, magic);
    if (!obj) {
        encode_string_u32(data, datapos, "");
        encode_u32(data, datapos, 0);
    } else {
        encode_string_u32(data, datapos, st->name);
        uint32_t p0 = *datapos;
        st->encode(st, NULL, datapos, obj); /* dry run: payload length */
        uint32_t length = *datapos - p0;
        *datapos = p0;
        encode_u32(data, datapos, length);
        st->encode(st, data, datapos, obj);
    }
    encode_u64(data, datapos, magic);
}

ASAM_API void *stype_decode_object(const uint8_t *data, uint32_t *datapos, uint32_t datalen, const stype_t **outstype)
{
    uint64_t magic = decode_u64(data, datapos, datalen);
    char *name = decode_string_u32(data, datapos, datalen);
    uint32_t length = decode_u32(data, datapos, datalen);
    void *obj = NULL;
    if (outstype)
        *outstype = NULL;
    stype_t *st = name ? stype_get(name) : NULL;
    if (st) {
        obj = st->decode(st, data, datapos, datalen);
        if (outstype)
            *outstype = st;
    } else if (length > 0) {
        /* unknown type: skip its payload (the length is part of the frame) */
        fprintf(stderr, "aprilsam_b200: unknown stype '%s' skipped (%u bytes)\n", name ? name : "?", length);
        if ((uint64_t) *datapos + length <= datalen)
            *datapos += length;
        else
            *datapos = datalen;
    }
    uint64_t magic2 = decode_u64(data, datapos, datalen);
    if (magic != magic2)
        asam_fatal("graph file: frame of '%s' is corrupt (magic %016" PRIx64 " vs %016" PRIx64 ")", name ? name : "?",
                   magic, magic2);
    free(name);
    return obj;
}

static int write_whole(const char *path, const uint8_t *buf, uint32_t len)
{
    FILE *f = fopen(path, "wb");
    if (!f)
        return -1;
    size_t w = fwrite(buf, 1, len, f);
    int rc = fclose(f);
    return (w == len && rc == 0) ? 0 : -1;
}

static uint8_t *read_whole(const char *path, uint32_t *len_out)
{
    FILE *f = fopen(path, "rb");
    if (!f)
        return NULL;
    fseek(f, 0L, SEEK_END);
    long len = ftell(f);
    fseek(f, 0L, SEEK_SET);
    if (len < 0 || (unsigned long) len > 0xffffffffUL) {
        fclose(f);
        return NULL;
    }
    uint8_t *buf = malloc((size_t) len + 1);
    size_t r = fread(buf, 1, (size_t) len, f);
    fclose(f);
    if (r != (size_t) len) {
        free(buf);
        return NULL;
    }
    *len_out = (uint32_t) len;
    return buf;
}

ASAM_API int stype_write_file(const stype_t *st, void *obj, const char *path)
{
    uint32_t len = 0;
    stype_encode_object(NULL, &len, st, obj);
    uint8_t *buf = calloc(1, (size_t) len + 1);
    len = 0;
    stype_encode_object(buf, &len, st, obj);
    int rc = write_whole(path, buf, len);
    free(buf);
    return rc;
}

ASAM_API void *stype_read_file(const char *path)
{
    uint32_t len = 0, pos = 0;
    uint8_t *buf = read_whole(path, &len);
    if (!buf)
        return NULL;
    void *obj = stype_decode_object(buf, &pos, len, NULL);
    free(buf);
    return obj;
}

/* ---- basic types (common/stype_basic_types.c) -------------------------------------------------- */
static void u64_encode(const stype_t *st, uint8_t *data, uint32_t *pos, const void *obj)
{
    (void) st;
    encode_u64(data, pos, *(const uint64_t *) obj);
}
static void *u64_decode(const stype_t *st, const uint8_t *data, uint32_t *pos, uint32_t len)
{
    (void) st;
    uint64_t *p = malloc(sizeof(uint64_t));
    *p = decode_u64(data, pos, len);
    return p;
}
static void *u64_copy(const stype_t *st, const void *obj)
{
    (void) st;
    uint64_t *p = malloc(sizeof(uint64_t));
    *p = *(const uint64_t *) obj;
    return p;
}
static void free_destroy(const stype_t *st, void *obj)
{
    (void) st;
    free(obj);
}
static void str_encode(const stype_t *st, uint8_t *data, uint32_t *pos, const void *obj)
{
    (void) st;
    encode_string_u32(data, pos, (const char *) obj);
}
static void *str_decode(const stype_t *st, const uint8_t *data, uint32_t *pos, uint32_t len)
{
    (void) st;
    return decode_string_u32(data, pos, len);
}
static void *str_copy(const stype_t *st, const void *obj)
{
    (void) st;
    return strdup((const char *) obj);
}

ASAM_API const stype_t stype_uint64 = { .name = "uint64", .encode = u64_encode, .decode = u64_decode, .copy = u64_copy,
                                        .destroy = free_destroy };
ASAM_API const stype_t stype_string = { .name = "string", .encode = str_encode, .decode = str_decode, .copy = str_copy,
                                        .destroy = free_destroy };

ASAM_API void stype_register_basic_types(void)
{
    stype_register(&stype_uint64);
    stype_register(&stype_string);
}

/* ---- attributes (april_graph.c:100-248) -------------------------------------------------------- */
typedef struct {
    char *key;
    const stype_t *stype;
    void *value;
} attr_rec_t;

typedef struct {
    attr_rec_t *rec;
    int n, cap;
} attr_table_t;

static void attr_encode(const stype_t *st, uint8_t *data, uint32_t *pos, const void *obj);
static void *attr_decode(const stype_t *st, const uint8_t *data, uint32_t *pos, uint32_t len);
static void *attr_copy(const stype_t *st, const void *obj);
static void attr_destroy_cb(const stype_t *st, void *obj);
ASAM_API const stype_t stype_april_graph_attr = { .name = "april_graph_attr_t", .encode = attr_encode,
                                                  .decode = attr_decode, .copy = attr_copy, .destroy = attr_destroy_cb };

ASAM_API april_graph_attr_t *april_graph_attr_create(void)
{
    april_graph_attr_t *a = calloc(1, sizeof(*a));
    a->stype = &stype_april_graph_attr;
    a->hash = (zhash_t *) calloc(1, sizeof(attr_table_t));
    return a;
}

ASAM_API void april_graph_attr_destroy(april_graph_attr_t *a)
{
    if (!a)
        return;
    attr_table_t *t = (attr_table_t *) a->hash;
    for (int i = 0; t && i < t->n; i++) {
        if (t->rec[i].value && t->rec[i].stype && t->rec[i].stype->destroy)
            t->rec[i].stype->destroy(t->rec[i].stype, t->rec[i].value);
        free(t->rec[i].key);
    }
    if (t)
        free(t->rec);
    free(t);
    free(a);
}

static void attr_put(april_graph_attr_t **pa, const stype_t *st, const char *key, void *value)
{
    if (!*pa)
        *pa = april_graph_attr_create();
    attr_table_t *t = (attr_table_t *) (*pa)->hash;
    for (int i = 0; i < t->n; i++)
        if (!strcmp(t->rec[i].key, key)) {
            /* like the reference, the caller stays responsible for a value it replaces */
            t->rec[i].stype = st;
            t->rec[i].value = value;
            return;
        }
    if (t->n == t->cap) {
        t->cap = t->cap ? 2 * t->cap : 4;
        t->rec = realloc(t->rec, sizeof(attr_rec_t) * (size_t) t->cap);
    }
    t->rec[t->n].key = strdup(key);
    t->rec[t->n].stype = st;
    t->rec[t->n].value = value;
    t->n++;
}

static void *attr_get(april_graph_attr_t *a, const char *key)
{
    if (!a)
        return NULL;
    attr_table_t *t = (attr_table_t *) a->hash;
    for (int i = 0; i < t->n; i++)
        if (!strcmp(t->rec[i].key, key))
            return t->rec[i].value;
    return NULL;
}

ASAM_API void april_graph_attr_put(april_graph_t *g, const stype_t *type, const char *key, void *data)
{
    attr_put(&g->attr, type, key, data);
}
ASAM_API void *april_graph_attr_get(april_graph_t *g, const char *key) { return attr_get(g->attr, key); }
ASAM_API void april_graph_factor_attr_put(april_graph_factor_t *f, const stype_t *type, const char *key, void *data)
{
    attr_put(&f->attr, type, key, data);
}
ASAM_API void *april_graph_factor_attr_get(april_graph_factor_t *f, const char *key) { return attr_get(f->attr, key); }
ASAM_API void april_graph_node_attr_put(april_graph_node_t *n, const stype_t *type, const char *key, void *data)
{
    attr_put(&n->attr, type, key, data);
}
ASAM_API void *april_graph_node_attr_get(april_graph_node_t *n, const char *key) { return attr_get(n->attr, key); }

/* april_graph.c:178-215: u8 1 | key | object ... u8 0; untyped values are not written */
static void attr_encode(const stype_t *st, uint8_t *data, uint32_t *pos, const void *obj)
{
    (void) st;
    const attr_table_t *t = (const attr_table_t *) ((const april_graph_attr_t *) obj)->hash;
    for (int i = 0; i < t->n; i++) {
        if (!t->rec[i].stype)
            continue;
        encode_u8(data, pos, 1);
        encode_string_u32(data, pos, t->rec[i].key);
        stype_encode_object(data, pos, t->rec[i].stype, t->rec[i].value);
    }
    encode_u8(data, pos, 0);
}

static void *attr_decode(const stype_t *st, const uint8_t *data, uint32_t *pos, uint32_t len)
{
    (void) st;
    april_graph_attr_t *a = april_graph_attr_create();
    while (decode_u8(data, pos, len)) {
        char *key = decode_string_u32(data, pos, len);
        const stype_t *vt = NULL;
        void *value = stype_decode_object(data, pos, len, &vt);
        if (key)
            attr_put(&a, vt, key, value);
        free(key);
    }
    return a;
}

/* deep copy of the values whose type can copy itself; others are dropped */
static void *attr_copy(const stype_t *st, const void *obj)
{
    (void) st;
    const attr_table_t *t = (const attr_table_t *) ((const april_graph_attr_t *) obj)->hash;
    april_graph_attr_t *a = april_graph_attr_create();
    for (int i = 0; i < t->n; i++) {
        const attr_rec_t *r = &t->rec[i];
        if (r->stype && r->stype->copy && r->value)
            attr_put(&a, r->stype, r->key, r->stype->copy(r->stype, r->value));
    }
    return a;
}

static void attr_destroy_cb(const stype_t *st, void *obj)
{
    (void) st;
    april_graph_attr_destroy((april_graph_attr_t *) obj);
}

april_graph_attr_t *asam_attr_dup(const april_graph_attr_t *a) { return a ? attr_copy(NULL, a) : NULL; }

/* ---- node / factor codecs (april_graph_xyt.c:216-269, :358-413; april_graph_xytpos.c:133-184) --- */
static void opt3_encode(uint8_t *data, uint32_t *pos, const double *v)
{
    encode_u8(data, pos, v ? 1 : 0);
    for (int i = 0; v && i < 3; i++)
        encode_f64(data, pos, v[i]);
}

static int opt3_decode(const uint8_t *data, uint32_t *pos, uint32_t len, double *v)
{
    if (!decode_u8(data, pos, len))
        return 0;
    for (int i = 0; i < 3; i++)
        v[i] = decode_f64(data, pos, len);
    return 1;
}

static void attr_of_encode(uint8_t *data, uint32_t *pos, const april_graph_attr_t *a)
{
    stype_encode_object(data, pos, a ? a->stype : NULL, a);
}

static void node_xyt_encode(const stype_t *st, uint8_t *data, uint32_t *pos, const void *obj)
{
    (void) st;
    const april_graph_node_t *n = obj;
    for (int i = 0; i < 3; i++)
        encode_f64(data, pos, n->state[i]);
    opt3_encode(data, pos, n->init);
    opt3_encode(data, pos, n->truth);
    attr_of_encode(data, pos, n->attr);
}

static void *node_xyt_decode(const stype_t *st, const uint8_t *data, uint32_t *pos, uint32_t len)
{
    (void) st;
    double state[3], init[3], truth[3];
    for (int i = 0; i < 3; i++)
        state[i] = decode_f64(data, pos, len);
    int hi = opt3_decode(data, pos, len, init), ht = opt3_decode(data, pos, len, truth);
    april_graph_node_t *n = april_graph_node_xyt_create(state, hi ? init : NULL, ht ? truth : NULL);
    n->attr = stype_decode_object(data, pos, len, NULL);
    return n;
}

/* xyt / xytpos: node ids | z | ztruth | W | attr.  The robust xyt factor (this library's own type) puts
 * u32 loss | f64 k between W and attr. */
static void factor_encode(const stype_t *st, uint8_t *data, uint32_t *pos, const void *obj)
{
    (void) st;
    const april_graph_factor_t *f = obj;
    for (int i = 0; i < f->nnodes; i++)
        encode_u32(data, pos, (uint32_t) f->nodes[i]);
    for (int i = 0; i < 3; i++)
        encode_f64(data, pos, f->u.common.z[i]);
    opt3_encode(data, pos, f->u.common.ztruth);
    for (int i = 0; i < 9; i++)
        encode_f64(data, pos, f->u.common.W->data[i]);
    if (f->type == APRIL_GRAPH_FACTOR_XYT_ROBUST_TYPE) {
        int32_t loss;
        double k;
        asam_factor_loss(f, &loss, &k);
        encode_u32(data, pos, (uint32_t) loss);
        encode_f64(data, pos, k);
    }
    attr_of_encode(data, pos, f->attr);
}

static void *factor_decode(const stype_t *st, const uint8_t *data, uint32_t *pos, uint32_t len)
{
    const int robust = st == &stype_april_factor_xyt_robust;
    const int binary = robust || !strcmp(st->name, "april_graph_factor_xyt");
    int a = (int) decode_u32(data, pos, len), b = binary ? (int) decode_u32(data, pos, len) : -1;
    double z[3], zt[3];
    for (int i = 0; i < 3; i++)
        z[i] = decode_f64(data, pos, len);
    int ht = opt3_decode(data, pos, len, zt); /* (the reference under-allocates ztruth here, quirk 15) */
    matd_t *W = matd_create(3, 3);
    for (int i = 0; i < 9; i++)
        W->data[i] = decode_f64(data, pos, len);
    april_graph_factor_t *f;
    if (robust) {
        int loss = (int) decode_u32(data, pos, len);
        double k = decode_f64(data, pos, len);
        f = aprilsam_b200_factor_xyt_robust_create(a, b, z, ht ? zt : NULL, W, loss, k);
        if (!f)
            asam_fatal("graph file: robust factor %d-%d: %s", a, b, aprilsam_b200_last_error());
    } else {
        f = binary ? april_graph_factor_xyt_create(a, b, z, ht ? zt : NULL, W)
                   : april_graph_factor_xytpos_create(a, z, ht ? zt : NULL, W);
    }
    f->attr = stype_decode_object(data, pos, len, NULL);
    matd_destroy(W);
    return f;
}

ASAM_API const stype_t stype_april_node_xyt = { .name = "april_graph_node_xyt", .encode = node_xyt_encode,
                                                .decode = node_xyt_decode };
ASAM_API const stype_t stype_april_factor_xyt = { .name = "april_graph_factor_xyt", .encode = factor_encode,
                                                  .decode = factor_decode };
ASAM_API const stype_t stype_april_factor_xytpos = { .name = "april_graph_factor_xytpos", .encode = factor_encode,
                                                     .decode = factor_decode };
ASAM_API const stype_t stype_april_factor_xyt_robust = { .name = "april_graph_factor_xyt_robust",
                                                         .encode = factor_encode, .decode = factor_decode };

/* ---- graph codec + files (april_graph.c:250-326, :377-426) ---------------------------------------- */
static void graph_encode(const stype_t *st, uint8_t *data, uint32_t *pos, const void *obj)
{
    (void) st;
    const april_graph_t *g = obj;
    for (int i = 0; i < zarray_size(g->nodes); i++) {
        april_graph_node_t *n;
        zarray_get(g->nodes, i, &n);
        if (!n->stype)
            continue; /* the reference prints "node without stype" and goes on */
        encode_u8(data, pos, 1);
        stype_encode_object(data, pos, n->stype, n);
    }
    for (int i = 0; i < zarray_size(g->factors); i++) {
        april_graph_factor_t *f;
        zarray_get(g->factors, i, &f);
        if (!f->stype)
            continue;
        encode_u8(data, pos, 2);
        stype_encode_object(data, pos, f->stype, f);
    }
    encode_u8(data, pos, 0);
    attr_of_encode(data, pos, g->attr);
}

static void *graph_decode(const stype_t *st, const uint8_t *data, uint32_t *pos, uint32_t len)
{
    (void) st;
    april_graph_t *g = april_graph_create();
    for (;;) {
        uint8_t op = decode_u8(data, pos, len);
        if (op == 0)
            break;
        if (op != 1 && op != 2)
            asam_fatal("graph file: bad opcode %d at byte %u", op, *pos);
        void *o = stype_decode_object(data, pos, len, NULL);
        if (o)
            zarray_add(op == 1 ? g->nodes : g->factors, &o);
    }
    g->attr = stype_decode_object(data, pos, len, NULL);
    return g;
}

ASAM_API const stype_t stype_april_graph = { .name = "april_graph_t", .encode = graph_encode, .decode = graph_decode };

ASAM_API void april_graph_stype_init(void)
{
    stype_register(&stype_april_graph);
    stype_register(&stype_april_graph_attr);
    stype_register(&stype_april_node_xyt);
    stype_register(&stype_april_factor_xyt);
    stype_register(&stype_april_factor_xytpos);
    stype_register(&stype_april_factor_xyt_robust);
}

/* returns 1 on success, 0 on failure (april_graph.c:377-398) */
ASAM_API int april_graph_save(april_graph_t *g, const char *path)
{
    uint32_t len = 0;
    stype_encode_object(NULL, &len, g->stype ? g->stype : &stype_april_graph, g);
    uint8_t *buf = malloc((size_t) len + 1);
    uint32_t pos = 0;
    stype_encode_object(buf, &pos, g->stype ? g->stype : &stype_april_graph, g);
    int rc = write_whole(path, buf, pos);
    free(buf);
    if (rc)
        printf("failed to open %s\n", path);
    return rc == 0;
}

/* NULL on failure (april_graph.c:400-426) */
ASAM_API april_graph_t *april_graph_create_from_file(const char *path)
{
    /* the built-in graph / node / factor types are registered on first use: the reference's
     * aprilsam_graph_save_simple.c forgets april_graph_stype_init() and dies in the reference's own
     * decoder (stype.c:163); here it loads */
    april_graph_stype_init();
    uint32_t len = 0, pos = 0;
    uint8_t *buf = read_whole(path, &len);
    if (!buf)
        return NULL;
    const stype_t *st = NULL;
    void *obj = stype_decode_object(buf, &pos, len, &st);
    free(buf);
    if (obj && st != &stype_april_graph) {
        fprintf(stderr, "aprilsam_b200: %s does not hold an april_graph_t\n", path);
        return NULL;
    }
    return obj;
}
