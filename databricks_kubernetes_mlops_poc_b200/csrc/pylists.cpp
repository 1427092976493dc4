/*
 * pylists.cpp -- the response side of the plugin call: C arrays -> Python lists, with recycled float objects.
 * Built into lib/libb2fpy.so (NOT into libb200forest.so, whose C ABI stays free of Python); loaded with ctypes.PyDLL,
 * i.e. every entry point runs with the GIL held.
 *
 * Reference counterpart: `self.classifier.predict_proba(...)[:, 1].tolist()` (databricks/src/02-register-model.ipynb:335-337):
 * the model object must hand plain Python lists to the handler (they are json.dumps'ed and re-validated, app/main.py:75-86).
 * At 65 536 rows that `.tolist()` -- one PyFloat allocation per element now, one free per element when the previous response
 * is dropped -- costs more than encoding, copying and scoring the whole batch (0.71 ms for the .tolist() alone against
 * 0.70 ms for a whole recycled-float predict() call, on the host of an H100 80GB HBM3 at 400 W), so the floats
 * are recycled: the module keeps a ring of float objects it owns one reference to; an object whose reference count is back
 * to 1 (nobody but the ring holds it: the response it was part of is gone) gets its value overwritten and goes into the
 * next list.  That is what CPython's own float free list does, at a larger scale; an object something else still
 * references is never touched (a fresh one takes its slot).  B200_FLOAT_POOL=0 turns the recycling off.
 */
#include <Python.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

namespace {
PyObject **g_ring = nullptr;
Py_ssize_t g_cap = 0, g_cursor = 0;
int g_enabled = -1;
long long g_reused = 0, g_fresh = 0;

bool pool_on() {
    if (g_enabled < 0) {
        const char *e = getenv("B200_FLOAT_POOL");
        g_enabled = (e && e[0] == '0') ? 0 : 1;
    }
    return g_enabled == 1;
}

bool pool_reserve(Py_ssize_t want) {
    /* room for three responses of this size: the one being built, the one the caller still holds, the one being dropped */
    const Py_ssize_t cap = want * 3 + 1024;
    if (cap <= g_cap) return true;
    if (cap > (Py_ssize_t)1 << 24) return false; /* 16 M floats (400 MB of objects): beyond that, plain allocation */
    PyObject **r = static_cast<PyObject **>(realloc(g_ring, (size_t)cap * sizeof(PyObject *)));
    if (!r) return false;
    memset(r + g_cap, 0, (size_t)(cap - g_cap) * sizeof(PyObject *));
    g_ring = r;
    g_cap = cap;
    return true;
}

inline PyObject *pooled_float(double v) {
    PyObject *&slot = g_ring[g_cursor];
    if (++g_cursor == g_cap) g_cursor = 0;
    PyObject *o = slot;
    if (o && Py_REFCNT(o) == 1) {
        reinterpret_cast<PyFloatObject *>(o)->ob_fval = v; /* nobody else can see this object */
        Py_SET_REFCNT(o, 2);                               /* the ring's reference + the list's */
        ++g_reused;
        return o;
    } else {
        o = PyFloat_FromDouble(v);
        if (!o) return nullptr;
        Py_XDECREF(slot); /* the old object lives on with whoever still references it */
        slot = o;
        ++g_fresh;
    }
    Py_INCREF(o);
    return o;
}
}  // namespace

extern "C" {

/* a list of n empty slots, to be filled by the *_fill_* calls before anything else sees it */
PyObject *b2f_py_list_new(Py_ssize_t n) { return PyList_New(n); }

/* items [offset, offset + n) of `list` <- float64 values at base, base + stride, ...; returns 0 / -1 (exception set) */
int b2f_py_list_fill_f64(PyObject *list, Py_ssize_t offset, const char *base, Py_ssize_t n, Py_ssize_t stride) {
    if (!PyList_CheckExact(list) || offset < 0 || n < 0 || offset + n > PyList_GET_SIZE(list)) {
        PyErr_SetString(PyExc_ValueError, "b2f_py_list_fill_f64: bad list or range");
        return -1;
    }
    const bool pooled = pool_on() && n >= 256 && pool_reserve(PyList_GET_SIZE(list));
    for (Py_ssize_t i = 0; i < n; ++i) {
        double v;
        memcpy(&v, base + i * stride, sizeof(v));
        PyObject *f = pooled ? pooled_float(v) : PyFloat_FromDouble(v);
        if (!f) return -1;
        PyObject *old = PyList_GET_ITEM(list, offset + i);
        PyList_SET_ITEM(list, offset + i, f);
        Py_XDECREF(old);
    }
    return 0;
}

/* the same for int32 values (outlier flags: 0 / 1 are interpreter singletons, no allocation) */
int b2f_py_list_fill_i32(PyObject *list, Py_ssize_t offset, const char *base, Py_ssize_t n, Py_ssize_t stride) {
    if (!PyList_CheckExact(list) || offset < 0 || n < 0 || offset + n > PyList_GET_SIZE(list)) {
        PyErr_SetString(PyExc_ValueError, "b2f_py_list_fill_i32: bad list or range");
        return -1;
    }
    for (Py_ssize_t i = 0; i < n; ++i) {
        int32_t v;
        memcpy(&v, base + i * stride, sizeof(v));
        PyObject *o = PyLong_FromLong(v);
        if (!o) return -1;
        PyObject *old = PyList_GET_ITEM(list, offset + i);
        PyList_SET_ITEM(list, offset + i, o);
        Py_XDECREF(old);
    }
    return 0;
}

/* (recycled, freshly allocated) float objects so far -- for tests and the bench breakdown */
void b2f_py_pool_stats(long long *reused, long long *fresh) {
    if (reused) *reused = g_reused;
    if (fresh) *fresh = g_fresh;
}

} /* extern "C" */
