"""Host-side mirror of the reference interface for the mxv/vxm + mxm path.

mxm with a mask is the int plus-times product of triangle counting (C takes the
mask's pattern); mxm(C, None, None, op, A, B, desc) is the unmasked sparse
product C = A (+.x) B for FP32 matrices over any order-independent semiring and
for INT32 matrices over PlusMultiplies.  eWiseAdd / eWiseMult with Matrix
operands are the union / intersection of two sparse matrices (FP32 over every
semiring, INT32 over PlusMultiplies), and transpose(C, None, None, A, desc) gives
C = A'.  With a sparse A and a dense FP32 B
(Matrix.build_dense / build_dense_device) the same call is SpMM: C becomes a dense
(nrows x ncols) matrix, read back with Matrix.extract_dense().

Classes and functions keep the reference's names, argument meaning and error
behaviour (every call returns/raises a graphblas::Info code):

  Descriptor   reference graphblas/descriptor.hpp:17-62
  Vector       reference graphblas/vector.hpp:13-264
  Matrix       reference graphblas/matrix.hpp:14-252
  vxm/mxv/mxm/eWiseAdd/eWiseMult/transpose/assign/reduce
               reference graphblas/operations.hpp:22-49,59-127,137-158,277-353,682-688,509-530,620-673

All compute goes through the C ABI (include/graphblast_b200.h); there is no
Python or CPU implementation of any operation here.
"""
import ctypes as C
import enum

import numpy as np

from . import _lib


class Info(enum.IntEnum):
    """reference graphblas/types.hpp:30-44"""
    GrB_SUCCESS = 0
    GrB_UNINITIALIZED_OBJECT = 1
    GrB_NULL_POINTER = 2
    GrB_INVALID_VALUE = 3
    GrB_INVALID_INDEX = 4
    GrB_DOMAIN_MISMATCH = 5
    GrB_DIMENSION_MISMATCH = 6
    GrB_OUTPUT_NOT_EMPTY = 7
    GrB_NO_VALUE = 8
    GrB_NOT_IMPLEMENTED = 9
    GrB_OUT_OF_MEMORY = 10
    GrB_INSUFFICIENT_SPACE = 11
    GrB_INVALID_OBJECT = 12
    GrB_INDEX_OUT_OF_BOUNDS = 13
    GrB_PANIC = 14


class Storage(enum.IntEnum):
    GrB_UNKNOWN = 0
    GrB_SPARSE = 1
    GrB_DENSE = 2


class Desc_field(enum.IntEnum):
    GrB_MASK = 0
    GrB_OUTP = 1
    GrB_INP0 = 2
    GrB_INP1 = 3
    GrB_MODE = 4
    GrB_TA = 5
    GrB_TB = 6
    GrB_NT = 7
    GrB_MXVMODE = 8
    GrB_TOL = 9
    GrB_BACKEND = 10


class Desc_value(enum.IntEnum):
    GrB_SCMP = 0
    GrB_REPLACE = 1
    GrB_TRAN = 2
    GrB_DEFAULT = 3
    GrB_PUSHPULL = 10
    GrB_PUSHONLY = 11
    GrB_PULLONLY = 12
    GrB_SEQUENTIAL = 13
    GrB_CUDA = 14


class GraphBLASError(RuntimeError):
    def __init__(self, info, what):
        self.info = Info(info)
        super().__init__("%s returned %s" % (what, self.info.name))


def _check(code, what):
    if code != 0:
        raise GraphBLASError(code, what)


class Semiring(enum.IntEnum):
    """REGISTER_SEMIRING order, reference graphblas/stddef.hpp:194-213"""
    LogicalOrAnd = 0
    PlusMultiplies = 1
    MinimumPlus = 2
    MaximumMultiplies = 3
    PlusDivides = 4
    PlusGreater = 5
    GreaterPlus = 6
    PlusMinus = 7
    PlusLess = 8
    CustomLessPlus = 9
    MinimumMultiplies = 10
    MultipliesMultiplies = 11
    NotEqualToPlus = 12
    MinimumSelectSecond = 13
    PlusNotEqualTo = 14
    CustomLessLess = 15
    MinimumNotEqualTo = 16


class Monoid(enum.IntEnum):
    """REGISTER_MONOID order, reference graphblas/stddef.hpp:160-173"""
    Plus = 0
    Multiplies = 1
    Minimum = 2
    Maximum = 3
    LogicalOr = 4
    LogicalAnd = 5
    Greater = 6
    CustomLess = 7
    NotEqualTo = 8


LogicalOrAndSemiring = Semiring.LogicalOrAnd
PlusMultipliesSemiring = Semiring.PlusMultiplies
MinimumPlusSemiring = Semiring.MinimumPlus
MaximumMultipliesSemiring = Semiring.MaximumMultiplies
PlusDividesSemiring = Semiring.PlusDivides
PlusGreaterSemiring = Semiring.PlusGreater
GreaterPlusSemiring = Semiring.GreaterPlus
PlusMinusSemiring = Semiring.PlusMinus
PlusLessSemiring = Semiring.PlusLess
CustomLessPlusSemiring = Semiring.CustomLessPlus
MinimumMultipliesSemiring = Semiring.MinimumMultiplies
MultipliesMultipliesSemiring = Semiring.MultipliesMultiplies
NotEqualToPlusSemiring = Semiring.NotEqualToPlus
MinimumSelectSecondSemiring = Semiring.MinimumSelectSecond
PlusNotEqualToSemiring = Semiring.PlusNotEqualTo
CustomLessLessSemiring = Semiring.CustomLessLess
MinimumNotEqualToSemiring = Semiring.MinimumNotEqualTo

PlusMonoid = Monoid.Plus
MultipliesMonoid = Monoid.Multiplies
MinimumMonoid = Monoid.Minimum
MaximumMonoid = Monoid.Maximum
LogicalOrMonoid = Monoid.LogicalOr
LogicalAndMonoid = Monoid.LogicalAnd
GreaterMonoid = Monoid.Greater
CustomLessMonoid = Monoid.CustomLess
NotEqualToMonoid = Monoid.NotEqualTo

FP32 = 0
INT32 = 1
_NP = {FP32: np.float32, INT32: np.int32}


def init(device=0):
    """One process per GPU: bind this process to `device`."""
    _check(_lib.load().gb200_init(int(device)), "gb200_init")


def sync():
    _check(_lib.load().gb200_sync(), "gb200_sync")


def sm_count():
    out = C.c_int(0)
    _check(_lib.load().gb200_sm_count(C.byref(out)), "gb200_sm_count")
    return out.value


def set_stream(cuda_stream_ptr):
    _check(_lib.load().gb200_set_stream(C.c_void_p(cuda_stream_ptr)),
           "gb200_set_stream")


def _ptr(arr):
    return arr.ctypes.data_as(C.c_void_p)


def _dev(t):
    """Device pointer of a torch tensor (or a raw int)."""
    if t is None:
        return None
    if isinstance(t, int):
        return C.c_void_p(t)
    return C.c_void_p(t.data_ptr())


class Descriptor(object):
    """graphblas::Descriptor.  Starts from the reference drivers' flag defaults
    (parseArgs, reference graphblas/util.hpp:39-132); keyword arguments set the
    same named knobs the command line does (mxvmode=0, struconly=1, ...)."""

    def __init__(self, **knobs):
        self._lib = _lib.load()
        h = C.c_void_p()
        _check(self._lib.gb200_desc_new(C.byref(h)), "Descriptor()")
        self._h = h
        for k, v in knobs.items():
            self.set_knob(k, v)

    def __del__(self):
        if getattr(self, "_h", None) is not None and self._h:
            self._lib.gb200_desc_free(self._h)
            self._h = None

    def set(self, field, value):
        _check(self._lib.gb200_desc_set(self._h, int(field), int(value)),
               "Descriptor::set")

    def get(self, field):
        out = C.c_int(0)
        _check(self._lib.gb200_desc_get(self._h, int(field), C.byref(out)),
               "Descriptor::get")
        try:
            return Desc_value(out.value)
        except ValueError:
            return out.value

    def toggle(self, field):
        _check(self._lib.gb200_desc_toggle(self._h, int(field)),
               "Descriptor::toggle")

    def set_knob(self, name, value):
        _check(self._lib.gb200_desc_set_knob(self._h, name.encode(),
                                             float(value)),
               "Descriptor knob %s" % name)

    def get_knob(self, name):
        out = C.c_double(0)
        _check(self._lib.gb200_desc_get_knob(self._h, name.encode(),
                                             C.byref(out)),
               "Descriptor knob %s" % name)
        return out.value

    @property
    def lastmxv(self):
        return Desc_value(int(self.get_knob("lastmxv")))


class Vector(object):
    """graphblas::Vector<float>."""

    def __init__(self, nsize, dtype=FP32):
        self._lib = _lib.load()
        self.dtype = dtype
        self._keep = []
        h = C.c_void_p()
        _check(self._lib.gb200_vector_new(C.byref(h), dtype, int(nsize)),
               "Vector(nsize)")
        self._h = h

    def __del__(self):
        if getattr(self, "_h", None) is not None and self._h:
            self._lib.gb200_vector_free(self._h)
            self._h = None

    # C API methods ---------------------------------------------------------
    def size(self):
        out = C.c_int(0)
        _check(self._lib.gb200_vector_size(self._h, C.byref(out)),
               "Vector::size")
        return out.value

    def nvals(self):
        out = C.c_int(0)
        _check(self._lib.gb200_vector_nvals(self._h, C.byref(out)),
               "Vector::nvals")
        return out.value

    def build(self, indices_or_values, values=None):
        """build(indices, values) -> sparse; build(values) -> dense (host data)."""
        if values is None:
            vals = np.ascontiguousarray(indices_or_values, dtype=np.float32)
            _check(self._lib.gb200_vector_build_dense(self._h, _ptr(vals),
                                                      len(vals)),
                   "Vector::build(values)")
        else:
            ind = np.ascontiguousarray(indices_or_values, dtype=np.int32)
            vals = np.ascontiguousarray(values, dtype=np.float32)
            _check(self._lib.gb200_vector_build_sparse(self._h, _ptr(ind),
                                                       _ptr(vals), len(ind)),
                   "Vector::build(indices, values)")

    def build_device(self, d_values, d_indices=None, nvals=None):
        """Adopt device memory (torch tensors); caller keeps ownership."""
        self._keep = [d_values, d_indices]
        if d_indices is None:
            n = d_values.numel() if nvals is None else nvals
            _check(self._lib.gb200_vector_adopt_dense(self._h, _dev(d_values), n),
                   "Vector::build(T*, nvals)")
        else:
            n = d_indices.numel() if nvals is None else nvals
            _check(self._lib.gb200_vector_adopt_sparse(self._h, _dev(d_indices),
                                                       _dev(d_values), n),
                   "Vector::build(Index*, T*, nvals)")

    def setElement(self, val, index):
        _check(self._lib.gb200_vector_set_element(self._h, float(val),
                                                  int(index)),
               "Vector::setElement")

    def extractTuples(self, sparse=False):
        """extractTuples(values, n): dense copy (sparse storage densified with 0);
        sparse=True returns (indices, values) of a sparse vector."""
        if sparse:
            n = C.c_int(self.size())
            ind = np.empty(n.value, dtype=np.int32)
            val = np.empty(n.value, dtype=np.float32)
            _check(self._lib.gb200_vector_extract_sparse(self._h, _ptr(ind),
                                                         _ptr(val),
                                                         C.byref(n)),
                   "Vector::extractTuples(indices, values)")
            return ind[:n.value].copy(), val[:n.value].copy()
        n = self.size()
        out = np.empty(n, dtype=np.float32)
        _check(self._lib.gb200_vector_extract_dense(self._h, _ptr(out), n),
               "Vector::extractTuples(values)")
        return out

    def extract_into(self, host_array):
        """extractTuples(values, n) into caller memory (e.g. pinned)."""
        n = self.size()
        if isinstance(host_array, np.ndarray):
            p = _ptr(host_array)
        else:
            p = C.c_void_p(host_array.data_ptr())
        _check(self._lib.gb200_vector_extract_dense(self._h, p, n),
               "Vector::extractTuples(values)")

    # handy methods ----------------------------------------------------------
    def fill(self, val):
        _check(self._lib.gb200_vector_fill(self._h, float(val)), "Vector::fill")

    def clear(self):
        _check(self._lib.gb200_vector_clear(self._h), "Vector::clear")

    def dup(self, rhs):
        _check(self._lib.gb200_vector_dup(self._h, rhs._h), "Vector::dup")

    def swap(self, rhs):
        """Trades contents with rhs, and with them the device tensors either one
        adopted (build_device), which must live as long as the contents do."""
        _check(self._lib.gb200_vector_swap(self._h, rhs._h), "Vector::swap")
        self._keep, rhs._keep = rhs._keep, self._keep

    def getStorage(self):
        out = C.c_int(0)
        _check(self._lib.gb200_vector_storage(self._h, C.byref(out)),
               "Vector::getStorage")
        return Storage(out.value)

    def sparse2dense(self, identity, desc=None):
        _check(self._lib.gb200_vector_sparse2dense(
            self._h, float(identity), desc._h if desc is not None else None),
            "Vector::sparse2dense")

    def dense2sparse(self, identity, desc):
        _check(self._lib.gb200_vector_dense2sparse(self._h, float(identity),
                                                   desc._h),
               "Vector::dense2sparse")

    def device_ptr(self):
        out = C.c_void_p()
        _check(self._lib.gb200_vector_device_ptr(self._h, C.byref(out)),
               "Vector device_ptr")
        return out.value


class Matrix(object):
    """graphblas::Matrix<float> (dtype FP32) or Matrix<int> (dtype INT32)."""

    def __init__(self, nrows=None, ncols=None, dtype=FP32, _handle=None):
        self._lib = _lib.load()
        self.dtype = dtype
        self._keep = []
        if _handle is not None:
            self._h = _handle
            return
        h = C.c_void_p()
        _check(self._lib.gb200_matrix_new(C.byref(h), dtype, int(nrows),
                                          int(ncols)),
               "Matrix(nrows, ncols)")
        self._h = h

    def __del__(self):
        if getattr(self, "_h", None) is not None and self._h:
            self._lib.gb200_matrix_free(self._h)
            self._h = None

    @classmethod
    def from_mtx(cls, path, directed=0, dtype=FP32):
        """readMtx + Matrix::build: the loader path of the reference drivers."""
        lib = _lib.load()
        h = C.c_void_p()
        _check(lib.gb200_matrix_load_mtx(C.byref(h), dtype, path.encode(),
                                         int(directed)),
               "readMtx/Matrix::build")
        return cls(dtype=dtype, _handle=h)

    def build(self, row_indices, col_indices, values=None, undirected=False):
        """Matrix::build from host COO triples."""
        r = np.ascontiguousarray(row_indices, dtype=np.int32)
        c = np.ascontiguousarray(col_indices, dtype=np.int32)
        v = None
        if values is not None:
            v = np.ascontiguousarray(values, dtype=_NP[self.dtype])
        _check(self._lib.gb200_matrix_build_coo(
            self._h, _ptr(r), _ptr(c), _ptr(v) if v is not None else None,
            len(r), 1 if undirected else 0), "Matrix::build(COO)")

    def build_device_csr(self, d_rowptr, d_colind, d_val, nvals,
                         d_colptr=None, d_rowind=None, d_cscval=None,
                         symmetric=False):
        """Matrix::build(Index* row_ptr, Index* col_ind, T* values, nvals) with
        DEVICE arrays (torch tensors), plus the CSC side."""
        self._keep = [d_rowptr, d_colind, d_val, d_colptr, d_rowind, d_cscval]
        _check(self._lib.gb200_matrix_adopt_csr(self._h, _dev(d_rowptr),
                                                _dev(d_colind), _dev(d_val),
                                                int(nvals)),
               "Matrix::build(device CSR)")
        _check(self._lib.gb200_matrix_adopt_csc(self._h, _dev(d_colptr),
                                                _dev(d_rowind), _dev(d_cscval),
                                                1 if symmetric else 0),
               "Matrix adopt CSC")

    def nrows(self):
        out = C.c_int(0)
        _check(self._lib.gb200_matrix_nrows(self._h, C.byref(out)),
               "Matrix::nrows")
        return out.value

    def ncols(self):
        out = C.c_int(0)
        _check(self._lib.gb200_matrix_ncols(self._h, C.byref(out)),
               "Matrix::ncols")
        return out.value

    def nvals(self):
        out = C.c_int(0)
        _check(self._lib.gb200_matrix_nvals(self._h, C.byref(out)),
               "Matrix::nvals")
        return out.value

    def extract_csr(self):
        """Host copy (rowptr, colind, val) of the CSR the CPU verifiers read."""
        n, nv = self.nrows(), self.nvals()
        rowptr = np.empty(n + 1, dtype=np.int32)
        colind = np.empty(max(nv, 1), dtype=np.int32)
        val = np.empty(max(nv, 1), dtype=_NP[self.dtype])
        _check(self._lib.gb200_matrix_extract_csr(self._h, _ptr(rowptr),
                                                  _ptr(colind), _ptr(val)),
               "Matrix extract CSR")
        return rowptr, colind[:nv], val[:nv]

    def build_dense(self, values):
        """Matrix::build(values, nvals): dense storage from a host array of shape
        (nrows, ncols), row-major (a flat array of fewer values leaves the rest 0)."""
        v = np.ascontiguousarray(values, dtype=np.float32)
        if v.ndim == 2 and v.shape != (self.nrows(), self.ncols()):
            raise ValueError("build_dense: shape %r, matrix is %d x %d" % (
                v.shape, self.nrows(), self.ncols()))
        _check(self._lib.gb200_matrix_build_dense(self._h, _ptr(v), v.size),
               "Matrix::build(values)")

    def build_dense_device(self, d_values):
        """Dense storage adopting a row-major float32 DEVICE tensor of at least
        nrows*ncols elements, read and written in place; the tensor is kept
        alive here and stays the caller's."""
        import torch
        need = self.nrows()*self.ncols()
        if d_values.dtype != torch.float32 or not d_values.is_contiguous() or \
                d_values.numel() < need:
            raise ValueError("build_dense_device: need a contiguous float32 tensor "
                             "of at least %d elements" % need)
        self._keep = [d_values]
        _check(self._lib.gb200_matrix_adopt_dense(self._h, _dev(d_values)),
               "Matrix adopt dense")

    def extract_dense(self):
        """Host copy of dense storage as an (nrows, ncols) float32 array."""
        out = np.empty((self.nrows(), self.ncols()), dtype=np.float32)
        _check(self._lib.gb200_matrix_extract_dense(self._h, _ptr(out), out.size),
               "Matrix::extractTuples(values)")
        return out

    def dense_ptr(self):
        out = C.c_void_p()
        _check(self._lib.gb200_matrix_dense_ptr(self._h, C.byref(out)),
               "Matrix dense_ptr")
        return out.value

    def getStorage(self):
        out = C.c_int(0)
        _check(self._lib.gb200_matrix_storage(self._h, C.byref(out)),
               "Matrix::getStorage")
        return Storage(out.value)

    def tril(self, desc):
        _check(self._lib.gb200_matrix_tril(self._h, desc._h), "tril")

    def apply_uniform_random(self, desc, seed, lo=1, hi=64):
        _check(self._lib.gb200_matrix_apply_uniform_random(self._h, desc._h,
                                                           int(seed), int(lo),
                                                           int(hi)),
               "apply(set_uniform_random)")

    def pr_normalize(self, alpha, desc):
        _check(self._lib.gb200_pr_normalize(self._h, float(alpha), desc._h),
               "PageRank normalisation")


def host_uniform_weights(seed, lo, hi, n):
    """The reference's SSSP weight stream (std::default_random_engine(seed),
    uniform_int[lo,hi]) into a host array; needs no device."""
    out = np.empty(n, dtype=np.float32)
    _check(_lib.load().gb200_host_uniform_weights(int(seed), int(lo), int(hi),
                                                  int(n), _ptr(out)),
           "host_uniform_weights")
    return out


def _h(obj):
    return obj._h if obj is not None else None


# Operations (argument order = reference graphblas/operations.hpp) ------------

def vxm(w, mask, accum, op, u, A, desc):
    _check(_lib.load().gb200_vxm(w._h, _h(mask), 0 if accum is None else 1,
                                 int(op), u._h, A._h, desc._h), "vxm")


def mxv(w, mask, accum, op, A, u, desc):
    _check(_lib.load().gb200_mxv(w._h, _h(mask), 0 if accum is None else 1,
                                 int(op), A._h, u._h, desc._h), "mxv")


def mxm(C_, mask, accum, op, A, B, desc):
    _check(_lib.load().gb200_mxm(C_._h, _h(mask), int(op), A._h, B._h, desc._h),
           "mxm")


def eWiseAdd(w, mask, accum, op, u, v, desc):
    """w = u + v.  With Matrix operands: the union of the two patterns, add(a, b)
    where both hold an entry, the one value where one does; C is replaced."""
    lib = _lib.load()
    if isinstance(w, Matrix):
        _check(lib.gb200_ewise_add_matrix(w._h, _h(mask), int(op), u._h, v._h,
                                          desc._h), "eWiseAdd(matrix)")
    elif isinstance(v, Vector):
        _check(lib.gb200_ewise_add(w._h, _h(mask), int(op), u._h, v._h,
                                   desc._h), "eWiseAdd")
    else:
        _check(lib.gb200_ewise_add_scalar(w._h, _h(mask), int(op), u._h,
                                          float(v), desc._h),
               "eWiseAdd(scalar)")


def eWiseMult(w, mask, accum, op, u, v, desc):
    """w = u .* v.  With Matrix operands: the intersection of the two patterns,
    mul(a, b); C is replaced."""
    lib = _lib.load()
    if isinstance(w, Matrix):
        _check(lib.gb200_ewise_mult_matrix(w._h, _h(mask), int(op), u._h, v._h,
                                           desc._h), "eWiseMult(matrix)")
    else:
        _check(lib.gb200_ewise_mult(w._h, _h(mask), int(op), u._h, v._h,
                                    desc._h), "eWiseMult")


def transpose(C_, mask, accum, A, desc):
    """C = A' (C = A when GrB_INP0 is GrB_TRAN); C may be A.  accum is not
    applied."""
    _check(_lib.load().gb200_transpose(C_._h, _h(mask), A._h, desc._h),
           "transpose")


def _indices(lst, n, what="extract"):
    """A host int32 array of an index list of at least n entries (kept alive by the
    caller), or None for GrB_ALL."""
    if lst is None:
        return None
    arr = np.ascontiguousarray(lst, dtype=np.int32).reshape(-1)
    if len(arr) < int(n):
        raise ValueError("%s: an index list of %d entries for a count of %d" % (
            what, len(arr), int(n)))
    return arr


def _ptr_or_null(arr):
    return None if arr is None else _ptr(arr)


def extract(out, mask, accum, src, rows, nrows, cols_or_col, ncols, desc):
    """Submatrix, column or subvector extract, in the reference's argument order.

    Matrix out: out = op(src)(rows, cols), cols_or_col a list, out nrows x ncols.
    Vector out, Matrix src: out = op(src)(rows, col), cols_or_col the column; ncols
    is ignored.  Vector out, Vector src: out = src(rows), of size nrows; cols_or_col
    and ncols are ignored.  op(src) is src' when desc's GrB_INP0 is GrB_TRAN.  None
    means GrB_ALL; lists are any int sequence or numpy array, sent as int32.  out is
    replaced: accum is not applied."""
    lib = _lib.load()
    r = _indices(rows, nrows)
    if isinstance(out, Matrix):
        c = _indices(cols_or_col, ncols)
        _check(lib.gb200_extract_matrix(out._h, _h(mask), src._h, _ptr_or_null(r),
                                        int(nrows), _ptr_or_null(c), int(ncols), desc._h),
               "extract(matrix)")
    elif isinstance(src, Matrix):
        _check(lib.gb200_extract_column(out._h, _h(mask), src._h, _ptr_or_null(r), int(nrows),
                                        int(cols_or_col), desc._h),
               "extract(column)")
    else:
        _check(lib.gb200_extract_vector(out._h, _h(mask), src._h, _ptr_or_null(r), int(nrows),
                                        desc._h),
               "extract(vector)")


NO_ACCUM = -1


def _accum_id(accum):
    """GB200_NO_ACCUM for None, otherwise the monoid's id."""
    return NO_ACCUM if accum is None else int(Monoid(accum))


def assign(out, mask, accum, src, *args):
    """Vector out: assign(w, mask, accum, val, indices, nindices, desc), w = val
    everywhere (indices must be None).

    Matrix out, in the reference's argument order (None means GrB_ALL; lists are any
    int sequence or numpy array, sent as int32, and may not repeat an index):
      assign(C, mask, accum, A_or_val, rows, nrows, cols, ncols, desc)
          C(rows, cols) = accum(C(rows, cols), op(A)), op(A) = A' when desc's
          GrB_INP0 is GrB_TRAN; or the scalar val at every position of the region;
      assign(C, mask, accum, u, rows, nrows, col, desc)   C(rows, col) = u;
      assign(C, mask, accum, u, row, cols, ncols, desc)   C(row, cols) = u.
    accum is None (C's region takes the source's pattern and values; C's entries in
    the region that the source does not store are deleted) or a Monoid (the union,
    accum(c, a) where both store an entry)."""
    lib = _lib.load()
    if not isinstance(out, Matrix):
        indices, nindices, desc = args
        if indices is not None:
            raise GraphBLASError(Info.GrB_NOT_IMPLEMENTED, "assign(indices)")
        _check(lib.gb200_assign_scalar(out._h, _h(mask), float(src), desc._h), "assign")
        return
    acc = _accum_id(accum)
    if len(args) == 5:
        rows, nrows, cols, ncols, desc = args
        r, c = _indices(rows, nrows, "assign"), _indices(cols, ncols, "assign")
        if isinstance(src, Matrix):
            _check(lib.gb200_assign_matrix(out._h, _h(mask), acc, src._h, _ptr_or_null(r),
                                           int(nrows), _ptr_or_null(c), int(ncols), desc._h),
                   "assign(matrix)")
        else:
            _check(lib.gb200_assign_matrix_scalar(out._h, _h(mask), acc, float(src),
                                                  _ptr_or_null(r), int(nrows), _ptr_or_null(c),
                                                  int(ncols), desc._h),
                   "assign(matrix, scalar)")
    elif len(args) == 4 and (args[0] is None or not np.isscalar(args[0])):
        rows, nrows, col, desc = args
        r = _indices(rows, nrows, "assign")
        _check(lib.gb200_assign_column(out._h, _h(mask), acc, src._h, _ptr_or_null(r),
                                       int(nrows), int(col), desc._h), "assign(column)")
    elif len(args) == 4:
        row, cols, ncols, desc = args
        c = _indices(cols, ncols, "assign")
        _check(lib.gb200_assign_row(out._h, _h(mask), acc, src._h, int(row), _ptr_or_null(c),
                                    int(ncols), desc._h), "assign(row)")
    else:
        raise TypeError("assign: %d arguments after the source" % len(args))


def reduce(accum, op, src, desc, out=None):
    """reduce(&val, accum, monoid, vector|matrix, desc) -> val
       reduce(.., out=w) for matrix rows -> vector w."""
    lib = _lib.load()
    if out is not None:
        _check(lib.gb200_reduce_matrix_rows(out._h, int(op), src._h, desc._h),
               "reduce(matrix rows)")
        return out
    val = C.c_double(0)
    if isinstance(src, Vector):
        _check(lib.gb200_reduce_vector(C.byref(val), int(op), src._h, desc._h),
               "reduce(vector)")
    else:
        _check(lib.gb200_reduce_matrix(C.byref(val), int(op), src._h, desc._h),
               "reduce(matrix)")
    return val.value
