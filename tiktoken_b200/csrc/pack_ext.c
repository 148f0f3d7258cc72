/*
 * pack_ext.c -- CPython helper for the host marshalling at the boundary ("next" row, SURVEY 8(f)-1):
 * list[str] -> one contiguous UTF-8 buffer + uint64 offsets, without creating a bytes object per
 * document.  The reference gets this for free because PyO3 borrows CPython's cached UTF-8
 * (`text: &str`, src/py.rs:30); here the batch has to be contiguous for ONE native call.
 * Pure host code (no CUDA); built by __graft_entry__.build() with gcc into tiktoken_b200/_b200pack*.so.
 */
#define _GNU_SOURCE
#define PY_SSIZE_T_CLEAN
#include <Python.h>
#include <stdint.h>
#include <string.h>
#include <unistd.h>

/* ---- pack(seq_of_str) -> (blob: bytes, offsets: bytes holding uint64[n+1]) ------------------------------------------
 * The strings are encoded to UTF-8 straight from CPython's compact representation (1 / 2 / 4 bytes per code point)
 * into their place of ONE blob, by a few threads: the calling thread collects (kind, data, length) of every string under
 * the GIL, the workers only READ those immutable buffers (no Python API off the calling thread; the list keeps the
 * strings alive, the caller waits).  ASCII strings are a memcpy.  str.encode semantics: a lone surrogate raises
 * UnicodeEncodeError (raised by CPython's own encoder on that item, so the exception is the canonical one).
 * (PyUnicode_AsUTF8AndSize would mean CPython's one-thread encoder plus a cached copy per string and a second memcpy.) */
#include <pthread.h>

typedef struct { const void *data; Py_ssize_t len; int kind; int ascii; } StrView;
typedef struct {
    const StrView *v; uint64_t *size_or_off; char *dst; Py_ssize_t lo, hi; Py_ssize_t bad;   /* bad: first item with a lone surrogate */
    int phase;
} PackJob;

#define UTF8_SIZE_LOOP(T)                                                                                        \
    { const T *p = (const T *)s->data; uint32_t sur = 0;                                                           \
      for (Py_ssize_t i = 0; i < s->len; i++) { const uint32_t c = p[i];                                            \
          n += 1u + (c >= 0x80u) + (c >= 0x800u) + (c >= 0x10000u); sur |= (uint32_t)(c - 0xD800u < 0x800u); }      \
      if (sur) *surrogate = 1; }
#define UTF8_WRITE_LOOP(T)                                                                                       \
    { const T *p = (const T *)s->data;                                                                             \
      for (Py_ssize_t i = 0; i < s->len; i++) { const uint32_t c = p[i];                                            \
          if (c < 0x80u) *d++ = (uint8_t)c;                                                                         \
          else if (c < 0x800u) { *d++ = (uint8_t)(0xC0 | (c >> 6)); *d++ = (uint8_t)(0x80 | (c & 0x3F)); }          \
          else if (c < 0x10000u) { *d++ = (uint8_t)(0xE0 | (c >> 12)); *d++ = (uint8_t)(0x80 | ((c >> 6) & 0x3F)); *d++ = (uint8_t)(0x80 | (c & 0x3F)); } \
          else { *d++ = (uint8_t)(0xF0 | (c >> 18)); *d++ = (uint8_t)(0x80 | ((c >> 12) & 0x3F)); *d++ = (uint8_t)(0x80 | ((c >> 6) & 0x3F)); *d++ = (uint8_t)(0x80 | (c & 0x3F)); } } }
static uint64_t utf8_size(const StrView *s, int *surrogate) {
    if (s->ascii) return (uint64_t)s->len;
    uint64_t n = 0;
    if (s->kind == 1) { const uint8_t *p = (const uint8_t *)s->data; for (Py_ssize_t i = 0; i < s->len; i++) n += 1u + (p[i] >> 7); }
    else if (s->kind == 2) UTF8_SIZE_LOOP(uint16_t)
    else UTF8_SIZE_LOOP(uint32_t)
    return n;
}
static void utf8_write(const StrView *s, uint8_t *d) {
    if (s->ascii) { memcpy(d, s->data, (size_t)s->len); return; }
    if (s->kind == 1) UTF8_WRITE_LOOP(uint8_t)
    else if (s->kind == 2) UTF8_WRITE_LOOP(uint16_t)
    else UTF8_WRITE_LOOP(uint32_t)
}
static void *pack_worker(void *arg) {
    PackJob *j = (PackJob *)arg;
    for (Py_ssize_t i = j->lo; i < j->hi; i++) {
        if (j->phase == 0) {
            int sur = 0;
            j->size_or_off[i] = utf8_size(&j->v[i], &sur);
            if (sur && j->bad < 0) j->bad = i;
        } else utf8_write(&j->v[i], (uint8_t *)j->dst + j->size_or_off[i]);
    }
    return NULL;
}
/* items [0, n) split into runs of about equal CODE POINT counts, one run per thread */
static void pack_run(PackJob *jobs, int nt, int phase) {
    pthread_t th[64];
    for (int t = 0; t < nt; t++) jobs[t].phase = phase;
    for (int t = 1; t < nt; t++) if (pthread_create(&th[t], NULL, pack_worker, &jobs[t]) != 0) { pack_worker(&jobs[t]); th[t] = 0; }
    pack_worker(&jobs[0]);
    for (int t = 1; t < nt; t++) if (th[t]) pthread_join(th[t], NULL);
}

static PyObject *pack(PyObject *self, PyObject *arg) {
    (void)self;
    PyObject *seq = PySequence_Fast(arg, "expected a sequence of str");
    if (!seq) return NULL;
    const Py_ssize_t n = PySequence_Fast_GET_SIZE(seq);
    PyObject **items = PySequence_Fast_ITEMS(seq);
    PyObject *offs = PyBytes_FromStringAndSize(NULL, (Py_ssize_t)((n + 1) * sizeof(uint64_t)));
    StrView *v = (StrView *)PyMem_Malloc((size_t)(n + 1) * sizeof(StrView));
    PyObject *blob = NULL;
    if (!offs || !v) { PyErr_NoMemory(); goto fail; }
    uint64_t *off = (uint64_t *)PyBytes_AS_STRING(offs);
    uint64_t total_cp = 0;
    for (Py_ssize_t i = 0; i < n; i++) {
        if (!PyUnicode_Check(items[i])) { PyErr_SetString(PyExc_TypeError, "expected str"); goto fail; }
        v[i].data = PyUnicode_DATA(items[i]); v[i].len = PyUnicode_GET_LENGTH(items[i]);
        v[i].kind = (int)PyUnicode_KIND(items[i]); v[i].ascii = PyUnicode_IS_ASCII(items[i]) ? 1 : 0;
        total_cp += (uint64_t)v[i].len;
    }
    {
        long ncpu = sysconf(_SC_NPROCESSORS_ONLN);
        int nt = (int)(total_cp >> 20);                            /* one thread per MiB of code points ... */
        if (nt > 16) nt = 16;
        if (ncpu > 0 && nt > ncpu) nt = (int)ncpu;                 /* ... up to 16 / the machine */
        if (nt < 1) nt = 1;
        PackJob jobs[64];
        Py_ssize_t lo = 0; uint64_t acc = 0;
        for (int t = 0; t < nt; t++) {
            const uint64_t want = total_cp / (uint64_t)nt * (uint64_t)(t + 1);
            Py_ssize_t hi = lo;
            if (t == nt - 1) hi = n; else while (hi < n && acc + (uint64_t)v[hi].len <= want) acc += (uint64_t)v[hi++].len;
            jobs[t].v = v; jobs[t].size_or_off = off; jobs[t].dst = NULL; jobs[t].lo = lo; jobs[t].hi = hi; jobs[t].bad = -1;
            lo = hi;
        }
        pack_run(jobs, nt, 0);                                     /* sizes */
        Py_ssize_t bad = -1;
        for (int t = 0; t < nt; t++) if (jobs[t].bad >= 0 && (bad < 0 || jobs[t].bad < bad)) bad = jobs[t].bad;
        if (bad >= 0) {                                            /* the canonical UnicodeEncodeError of that string */
            Py_ssize_t len;
            if (PyUnicode_AsUTF8AndSize(items[bad], &len)) PyErr_SetString(PyExc_UnicodeEncodeError, "surrogates not allowed");
            goto fail;
        }
        uint64_t total = 0;
        for (Py_ssize_t i = 0; i < n; i++) { const uint64_t sz = off[i]; off[i] = total; total += sz; }
        off[n] = total;
        blob = PyBytes_FromStringAndSize(NULL, (Py_ssize_t)total);
        if (!blob) goto fail;
        for (int t = 0; t < nt; t++) jobs[t].dst = PyBytes_AS_STRING(blob);
        pack_run(jobs, nt, 1);                                     /* bytes */
    }
    PyMem_Free(v);
    Py_DECREF(seq);
    return Py_BuildValue("(NN)", blob, offs);
fail:
    PyMem_Free(v);
    Py_XDECREF(offs); Py_DECREF(seq);
    return NULL;
}

/* unpack(tokens_addr: int, offsets_addr: int, n_docs: int[, int_cache: list]) -> list[list[int]]
 * The reference converts Vec<Vec<Rank>> into Python lists of freshly made int objects (PyO3); making ~230 M ints per GiB
 * of text is what bounds the list-returning batch API on both sides.  Token ids come from a vocabulary of
 * 50-200 k entries, so the int OBJECTS can be shared: `int_cache[i] is i` for every id, built once per encoding -- a token
 * then costs one table load and one reference count instead of an allocation. */
static PyObject *unpack(PyObject *self, PyObject *args) {
    (void)self;
    unsigned long long ta, oa; Py_ssize_t n; PyObject *cache = NULL;
    if (!PyArg_ParseTuple(args, "KKn|O", &ta, &oa, &n, &cache)) return NULL;
    const uint32_t *tok = (const uint32_t *)(uintptr_t)ta;
    const uint64_t *off = (const uint64_t *)(uintptr_t)oa;
    PyObject **citems = NULL; Py_ssize_t clen = 0;
    if (cache && cache != Py_None) {
        if (!PyList_CheckExact(cache)) { PyErr_SetString(PyExc_TypeError, "int_cache must be a list"); return NULL; }
        citems = PySequence_Fast_ITEMS(cache); clen = PyList_GET_SIZE(cache);
    }
    PyObject *out = PyList_New(n);
    if (!out) return NULL;
    for (Py_ssize_t d = 0; d < n; d++) {
        const uint64_t lo = off[d], hi = off[d + 1];
        PyObject *doc = PyList_New((Py_ssize_t)(hi - lo));
        if (!doc) { Py_DECREF(out); return NULL; }
        for (uint64_t k = lo; k < hi; k++) {
            const uint32_t t = tok[k];
            PyObject *v;
            if ((Py_ssize_t)t < clen) { v = citems[t]; Py_INCREF(v); }
            else {
                v = PyLong_FromUnsignedLong(t);
                if (!v) { Py_DECREF(doc); Py_DECREF(out); return NULL; }
            }
            PyList_SET_ITEM(doc, (Py_ssize_t)(k - lo), v);
        }
        PyList_SET_ITEM(out, d, doc);
    }
    return out;
}


/* find_first(blob, offsets, needles) -> None | (doc, needle_index, byte_pos)
 * The disallowed-special check of tiktoken/core.py:120-124 on the PACKED batch: the first document (in order)
 * that contains any of the byte strings `needles`, and the leftmost occurrence in it (longest on ties).  A match
 * never straddles two documents.  One memchr pass when all needles share their first byte (they do for the
 * published encodings: "<|"), else one memmem pass per needle. */
static PyObject *find_first(PyObject *self, PyObject *args) {
    (void)self;
    Py_buffer blob, offs;
    PyObject *needles_obj;
    if (!PyArg_ParseTuple(args, "y*y*O", &blob, &offs, &needles_obj)) return NULL;
    PyObject *seq = PySequence_Fast(needles_obj, "needles must be a sequence of bytes");
    if (!seq) { PyBuffer_Release(&blob); PyBuffer_Release(&offs); return NULL; }
    const Py_ssize_t nn = PySequence_Fast_GET_SIZE(seq);
    const char **np_ = (const char **)PyMem_Malloc((size_t)(nn + 1) * sizeof(char *));
    Py_ssize_t *nl = (Py_ssize_t *)PyMem_Malloc((size_t)(nn + 1) * sizeof(Py_ssize_t));
    PyObject *ret = NULL;
    int same_first = 1;
    for (Py_ssize_t a = 0; a < nn; a++) {
        char *p; Py_ssize_t l;
        if (PyBytes_AsStringAndSize(PySequence_Fast_GET_ITEM(seq, a), &p, &l) < 0) goto done;
        np_[a] = p; nl[a] = l;
        if (l == 0) { PyErr_SetString(PyExc_ValueError, "empty needle"); goto done; }
        if (p[0] != np_[0][0]) same_first = 0;
    }
    {
        const uint8_t *text = (const uint8_t *)blob.buf;
        const uint64_t *off = (const uint64_t *)offs.buf;
        const Py_ssize_t n_docs = offs.len / 8 - 1;
        for (Py_ssize_t d = 0; d < n_docs; d++)
            if (off[d] > off[d + 1] || off[d + 1] > (uint64_t)blob.len) {
                PyErr_SetString(PyExc_ValueError, "offsets must be non-decreasing and end inside the blob");
                goto done;
            }
        Py_ssize_t hit_doc = -1, hit_a = -1; uint64_t hit_pos = 0;
        Py_BEGIN_ALLOW_THREADS
        for (Py_ssize_t d = 0; d < n_docs && hit_doc < 0 && nn > 0; d++) {
            const uint8_t *s = text + off[d], *e = text + off[d + 1];
            const uint8_t *best = NULL; Py_ssize_t best_a = -1;
            if (same_first) {
                const uint8_t *p = s;
                while (!best && p < e && (p = (const uint8_t *)memchr(p, np_[0][0], (size_t)(e - p))) != NULL) {
                    for (Py_ssize_t a = 0; a < nn; a++)
                        if (nl[a] <= e - p && memcmp(p, np_[a], (size_t)nl[a]) == 0 && (best_a < 0 || nl[a] > nl[best_a])) { best = p; best_a = a; }
                    p++;
                }
            } else {
                for (Py_ssize_t a = 0; a < nn; a++) {
                    if (nl[a] > e - s) continue;
                    const uint8_t *f = (const uint8_t *)memmem(s, (size_t)(e - s), np_[a], (size_t)nl[a]);
                    if (f && (!best || f < best || (f == best && nl[a] > nl[best_a]))) { best = f; best_a = a; }
                }
            }
            if (best) { hit_doc = d; hit_a = best_a; hit_pos = (uint64_t)(best - text); }
        }
        Py_END_ALLOW_THREADS
        if (hit_doc < 0) { ret = Py_None; Py_INCREF(ret); }
        else ret = Py_BuildValue("(nnK)", hit_doc, hit_a, (unsigned long long)hit_pos);
    }
done:
    PyMem_Free(np_); PyMem_Free(nl);
    Py_DECREF(seq); PyBuffer_Release(&blob); PyBuffer_Release(&offs);
    return ret;
}


/* parse_tiktoken(data: bytes) -> (blob: bytes, offsets: bytes uint64[n+1], ranks: bytes uint32[n])
 * The `.tiktoken` vocabulary format of tiktoken/load.py:159-171 -- one "base64(token) rank" line per token --
 * straight into the flattened arrays b200bpe_create takes, without a Python dict of 100-200 k bytes objects. */
static PyObject *parse_tiktoken(PyObject *self, PyObject *arg) {
    (void)self;
    Py_buffer in;
    if (PyObject_GetBuffer(arg, &in, PyBUF_SIMPLE) < 0) return NULL;
    const unsigned char *p = (const unsigned char *)in.buf, *end = p + in.len;
    signed char dec[256];
    memset(dec, -1, sizeof dec);
    for (int i = 0; i < 26; i++) { dec['A' + i] = (signed char)i; dec['a' + i] = (signed char)(26 + i); }
    for (int i = 0; i < 10; i++) dec['0' + i] = (signed char)(52 + i);
    dec['+'] = 62; dec['/'] = 63;
    size_t n_lines = 0;
    for (const unsigned char *q = p; q < end; q++) n_lines += (*q == '\n');
    n_lines += 1;
    unsigned char *blob = (unsigned char *)PyMem_Malloc((size_t)in.len + 4);       /* decoded bytes < input bytes */
    uint64_t *off = (uint64_t *)PyMem_Malloc((n_lines + 1) * sizeof(uint64_t));
    uint32_t *rank = (uint32_t *)PyMem_Malloc((n_lines + 1) * sizeof(uint32_t));
    PyObject *ret = NULL;
    if (!blob || !off || !rank) { PyErr_NoMemory(); goto done; }
    {
        size_t n = 0, nb = 0;
        while (p < end) {
            const unsigned char *eol = (const unsigned char *)memchr(p, '\n', (size_t)(end - p));
            if (!eol) eol = end;
            const unsigned char *le = eol;
            if (le > p && le[-1] == '\r') le--;
            if (le == p) { p = eol + 1; continue; }                                   /* empty line (load.py:165) */
            const unsigned char *sp = (const unsigned char *)memchr(p, ' ', (size_t)(le - p));
            if (!sp || sp == p || sp + 1 >= le) { PyErr_Format(PyExc_ValueError, "malformed line %zu", n + 1); goto done; }
            off[n] = nb;
            uint32_t acc = 0; int bits = 0;
            const unsigned char *q = p;
            for (; q < sp && *q != '='; q++) {
                const int v = dec[*q];
                if (v < 0) { PyErr_Format(PyExc_ValueError, "bad base64 on line %zu", n + 1); goto done; }
                acc = (acc << 6) | (uint32_t)v; bits += 6;
                if (bits >= 8) { bits -= 8; blob[nb++] = (unsigned char)(acc >> bits); acc &= (1u << bits) - 1u; }
            }
            for (; q < sp; q++) if (*q != '=') { PyErr_Format(PyExc_ValueError, "bad base64 padding on line %zu", n + 1); goto done; }
            if (nb == off[n]) { PyErr_Format(PyExc_ValueError, "empty token on line %zu", n + 1); goto done; }
            uint64_t r = 0;
            for (q = sp + 1; q < le; q++) {
                if (*q < '0' || *q > '9') { PyErr_Format(PyExc_ValueError, "bad rank on line %zu", n + 1); goto done; }
                r = r * 10 + (uint64_t)(*q - '0');
                if (r > 0xFFFFFFFFull) { PyErr_Format(PyExc_ValueError, "rank too large on line %zu", n + 1); goto done; }
            }
            rank[n++] = (uint32_t)r;
            p = eol + 1;
        }
        off[n] = nb;
        ret = Py_BuildValue("(y#y#y#)", (const char *)blob, (Py_ssize_t)nb, (const char *)off, (Py_ssize_t)((n + 1) * sizeof(uint64_t)),
                            (const char *)rank, (Py_ssize_t)(n * sizeof(uint32_t)));
    }
done:
    PyMem_Free(blob); PyMem_Free(off); PyMem_Free(rank);
    PyBuffer_Release(&in);
    return ret;
}

static PyMethodDef methods[] = {
    {"pack", pack, METH_O, "list[str] -> (utf8 blob bytes, uint64 offsets bytes)"},
    {"unpack", unpack, METH_VARARGS, "(tokens_addr, offsets_addr, n_docs) -> list[list[int]]"},
    {"parse_tiktoken", parse_tiktoken, METH_O, "(.tiktoken file bytes) -> (blob, offsets uint64, ranks uint32)"},
    {"find_first", find_first, METH_VARARGS, "(blob, offsets, needles) -> None | (doc, needle_index, byte_pos)"},
    {NULL, NULL, 0, NULL}};
static struct PyModuleDef mod = {PyModuleDef_HEAD_INIT, "_b200pack", "host marshalling helpers", -1, methods, NULL, NULL, NULL, NULL};
PyMODINIT_FUNC PyInit__b200pack(void) { return PyModule_Create(&mod); }
