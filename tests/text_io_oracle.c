/* A CPU restatement of vector_in / halfvec_in / sparsevec_in (src/vector.c:174-281, src/halfvec.c:178-286,
 * src/sparsevec.c:203-409) over glibc strtof / strtol in the C locale, for the tests of the device type I/O.
 * Each function returns 0 and the row, or 1 with the reference's errmsg / errdetail. TEST INFRASTRUCTURE ONLY. */
#include <errno.h>
#include <limits.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define MAXDIM 16000
#define MSG 300000

static int sp(char c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r' || c == '\v' || c == '\f'; }

static int fail(char *msg, char *detail, const char *d, const char *fmt, const char *a, const char *b) {
    snprintf(msg, MSG, fmt, a, b);
    strcpy(detail, d ? d : "");
    return 1;
}

static uint16_t to_half(float f, int *inf) {
    _Float16 h = (_Float16)f;
    uint16_t u;
    memcpy(&u, &h, 2);
    *inf = (u & 0x7fff) == 0x7c00;
    return u;
}

/* half = 0: vector (float out), 1: halfvec (uint16 out) */
int text_dense_in(int half, const char *lit, int32_t typmod, void *out, int *dim_out, char *msg, char *detail) {
    const char *t = half ? "halfvec" : "vector";
    const char *pt = lit;
    int dim = 0;
    char tmp[128];
    while (sp(*pt)) pt++;
    if (*pt != '[') return fail(msg, detail, "Vector contents must start with \"[\".", "invalid input syntax for type %s: \"%s\"", t, lit);
    pt++;
    while (sp(*pt)) pt++;
    if (*pt == ']') return fail(msg, detail, NULL, "%s must have at least 1 dimension%s", t, "");
    for (;;) {
        char *end;
        float val;
        if (dim == MAXDIM) { snprintf(tmp, sizeof tmp, "%d", MAXDIM); return fail(msg, detail, NULL, "%s cannot have more than %s dimensions", t, tmp); }
        while (sp(*pt)) pt++;
        if (*pt == '\0') return fail(msg, detail, NULL, "invalid input syntax for type %s: \"%s\"", t, lit);
        errno = 0;
        val = strtof(pt, &end);
        if (end == pt) return fail(msg, detail, NULL, "invalid input syntax for type %s: \"%s\"", t, lit);
        if (half) {
            int hinf;
            uint16_t h = to_half(val, &hinf);
            if ((errno == ERANGE && isinf(val)) || (hinf && !isinf(val))) {
                char *tok = strndup(pt, (size_t)(end - pt));
                snprintf(msg, MSG, "\"%s\" is out of range for type %s", tok, t);
                free(tok);
                detail[0] = 0;
                return 1;
            }
            if ((h & 0x7fff) > 0x7c00) return fail(msg, detail, NULL, "NaN not allowed in %s%s", t, "");
            if (hinf) return fail(msg, detail, NULL, "infinite value not allowed in %s%s", t, "");
            ((uint16_t *)out)[dim++] = h;
        } else {
            if (errno == ERANGE && isinf(val)) {
                char *tok = strndup(pt, (size_t)(end - pt));
                snprintf(msg, MSG, "\"%s\" is out of range for type %s", tok, t);
                free(tok);
                detail[0] = 0;
                return 1;
            }
            if (isnan(val)) return fail(msg, detail, NULL, "NaN not allowed in %s%s", t, "");
            if (isinf(val)) return fail(msg, detail, NULL, "infinite value not allowed in %s%s", t, "");
            ((float *)out)[dim++] = val;
        }
        pt = end;
        while (sp(*pt)) pt++;
        if (*pt == ',') pt++;
        else if (*pt == ']') { pt++; break; }
        else return fail(msg, detail, NULL, "invalid input syntax for type %s: \"%s\"", t, lit);
    }
    while (sp(*pt)) pt++;
    if (*pt != '\0') return fail(msg, detail, "Junk after closing right brace.", "invalid input syntax for type %s: \"%s\"", t, lit);
    if (typmod != -1 && typmod != dim) { snprintf(msg, MSG, "expected %d dimensions, not %d", typmod, dim); detail[0] = 0; return 1; }
    *dim_out = dim;
    return 0;
}

typedef struct { int32_t index; float value; } Elem;
static int cmp_elem(const void *a, const void *b) {
    int32_t x = ((const Elem *)a)->index, y = ((const Elem *)b)->index;
    return x < y ? -1 : x > y;
}

int text_sparse_in(const char *lit, int32_t typmod, int32_t *idx, float *val, int *nnz_out, int *dim_out, char *msg, char *detail) {
    const char *t = "sparsevec";
    const char *pt = lit;
    int max_nnz = 1, nnz = 0, dim;
    long ldim;
    char *end;
    Elem *el;
    for (const char *q = lit; *q; q++) max_nnz += *q == ',';
    if (max_nnz > MAXDIM) return fail(msg, detail, NULL, "sparsevec cannot have more than %s non-zero elements%s", "16000", "");
    el = malloc(sizeof(Elem) * (size_t)max_nnz);
    while (sp(*pt)) pt++;
    if (*pt != '{') { free(el); return fail(msg, detail, "Vector contents must start with \"{\".", "invalid input syntax for type %s: \"%s\"", t, lit); }
    pt++;
    while (sp(*pt)) pt++;
    if (*pt == '}') pt++;
    else for (;;) {
        long index;
        float value;
        while (sp(*pt)) pt++;
        if (*pt == '\0') goto syntax;
        index = strtol(pt, &end, 10);
        if (end == pt) goto syntax;
        if (index > INT_MAX) index = INT_MAX;
        else if (index < INT_MIN + 1) index = INT_MIN + 1;
        pt = end;
        while (sp(*pt)) pt++;
        if (*pt != ':') goto syntax;
        pt++;
        while (sp(*pt)) pt++;
        errno = 0;
        value = strtof(pt, &end);
        if (end == pt) goto syntax;
        if (errno == ERANGE && (value == 0 || isinf(value))) {
            char *tok = strndup(pt, (size_t)(end - pt));
            snprintf(msg, MSG, "\"%s\" is out of range for type %s", tok, t);
            free(tok);
            detail[0] = 0;
            free(el);
            return 1;
        }
        if (isnan(value)) { free(el); return fail(msg, detail, NULL, "NaN not allowed in %s%s", t, ""); }
        if (isinf(value)) { free(el); return fail(msg, detail, NULL, "infinite value not allowed in %s%s", t, ""); }
        if (value != 0) { el[nnz].index = (int32_t)(index - 1); el[nnz].value = value; nnz++; }
        pt = end;
        while (sp(*pt)) pt++;
        if (*pt == ',') pt++;
        else if (*pt == '}') { pt++; break; }
        else goto syntax;
    }
    while (sp(*pt)) pt++;
    if (*pt != '/') { free(el); return fail(msg, detail, "Unexpected end of input.", "invalid input syntax for type %s: \"%s\"", t, lit); }
    pt++;
    while (sp(*pt)) pt++;
    ldim = strtol(pt, &end, 10);
    if (end == pt) goto syntax;
    if (ldim > INT_MAX) ldim = INT_MAX;
    else if (ldim < INT_MIN) ldim = INT_MIN;
    dim = (int)ldim;
    pt = end;
    while (sp(*pt)) pt++;
    if (*pt != '\0') { free(el); return fail(msg, detail, "Junk after closing.", "invalid input syntax for type %s: \"%s\"", t, lit); }
    if (dim < 1) { free(el); return fail(msg, detail, NULL, "sparsevec must have at least 1 dimension%s%s", "", ""); }
    if (dim > 1000000000) { free(el); return fail(msg, detail, NULL, "sparsevec cannot have more than %s dimensions%s", "1000000000", ""); }
    if (typmod != -1 && typmod != dim) { snprintf(msg, MSG, "expected %d dimensions, not %d", typmod, dim); detail[0] = 0; free(el); return 1; }
    qsort(el, (size_t)nnz, sizeof(Elem), cmp_elem);
    for (int i = 0; i < nnz; i++) {
        idx[i] = el[i].index;
        val[i] = el[i].value;
        if (idx[i] < 0 || idx[i] >= dim) { free(el); return fail(msg, detail, NULL, "sparsevec index out of bounds%s%s", "", ""); }
        if (i > 0 && idx[i] == idx[i - 1]) { free(el); return fail(msg, detail, NULL, "sparsevec indices must not contain duplicates%s%s", "", ""); }
    }
    free(el);
    *nnz_out = nnz;
    *dim_out = dim;
    return 0;
syntax:
    free(el);
    return fail(msg, detail, NULL, "invalid input syntax for type %s: \"%s\"", t, lit);
}

/* strtof in the C locale: the value's bits, the end offset and errno == ERANGE */
uint32_t text_strtof(const char *s, int *end, int *erange) {
    char *e;
    float f;
    uint32_t u;
    errno = 0;
    f = strtof(s, &e);
    *erange = errno == ERANGE;
    *end = (int)(e - s);
    memcpy(&u, &f, 4);
    return u;
}
