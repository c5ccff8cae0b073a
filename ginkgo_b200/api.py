"""Python face of the library, mirroring the reference's operator interface for the
hot path (same names, argument meaning and error behaviour):

    exec = B200Executor.create(0)                 # gko::CudaExecutor::create
    A = Csr.create(exec, (n, m), values, col_idxs, row_ptrs)   # gko::matrix::Csr::create
    A.apply(b, x)                                 # LinOp::apply(b, x):          x = A b
    A.apply(alpha, b, beta, x)                    # LinOp::apply(alpha,b,beta,x) x = aAb + bx

Device memory and streams come from torch (plumbing); every computation goes through the
C ABI of include/ginkgo_b200.h into hand-written sm_90a kernels.  Operands that live on the
host are cloned to the executor for the call and the result copied back, exactly like
LinOp::apply's make_temporary_clone (include/ginkgo/core/base/lin_op.hpp:129-215).
There is no CPU fallback."""
import ctypes

import torch

from . import _lib

_VT = {torch.float64: "f64", torch.float32: "f32"}
_IT = {torch.int32: "i32", torch.int64: "i64"}


class DimensionMismatch(ValueError):
    """gko::DimensionMismatch"""


class NotSupported(TypeError):
    """gko::NotSupported"""


class B200Executor:
    """gko::CudaExecutor analogue: one device + one stream + the C-ABI context."""

    def __init__(self, device_id, stream):
        self.device_id = device_id
        self.device = torch.device("cuda", device_id)
        self.stream = stream
        self._l = _lib.lib()
        ctx = ctypes.c_void_p()
        _lib.check(self._l.b200_ctx_create(device_id, stream.cuda_stream, ctypes.byref(ctx)))
        self.ctx = ctx

    @staticmethod
    def create(device_id=0, stream=None):
        if not torch.cuda.is_available():
            raise _lib.B200Error("B200Executor needs a CUDA device (no CPU fallback)")
        with torch.cuda.device(device_id):
            stream = stream or torch.cuda.Stream(device_id)
        return B200Executor(device_id, stream)

    def synchronize(self):
        _lib.check(self._l.b200_synchronize(self.ctx))

    def launch_count(self):
        return self._l.b200_ctx_launch_count(self.ctx)

    def num_sms(self):
        return self._l.b200_ctx_num_sms(self.ctx)

    def run(self, name, *args):
        """exec->run(make_<op>(...)): enqueue one C-ABI call on the executor's stream"""
        _lib.call(name, self.ctx, *args)

    def __del__(self):
        try:
            self._l.b200_ctx_destroy(self.ctx)
        except Exception:
            pass


class Dense:
    """gko::matrix::Dense: row-major values with a row stride."""

    def __init__(self, exec_, values, size=None, stride=None):
        if values.dim() == 1:
            values = values.reshape(-1, 1)
        self.exec = exec_
        self.values = values
        self.size = tuple(size) if size is not None else tuple(values.shape)
        self.stride = stride if stride is not None else values.stride(0) if values.shape[0] > 1 \
            else values.shape[1]
        if values.dtype not in _VT:
            raise NotSupported("value type %s" % values.dtype)

    @staticmethod
    def create(exec_, size, values=None, stride=None, dtype=torch.float64):
        rows, cols = size
        stride = cols if stride is None else stride
        if values is None:
            with torch.cuda.stream(exec_.stream):
                values = torch.empty((rows, stride), dtype=dtype, device=exec_.device)
        return Dense(exec_, values, (rows, cols), stride)

    @property
    def vt(self):
        return _VT[self.values.dtype]

    @property
    def on_device(self):
        return self.values.is_cuda

    def to_device(self, exec_):
        if self.on_device:
            return self
        with torch.cuda.stream(exec_.stream):
            v = self.values.to(exec_.device, non_blocking=True)
        return Dense(exec_, v, self.size, self.stride)


class _SparseBase:
    def _check(self, b, x):
        if b.size[0] != self.size[1] or x.size[0] != self.size[0] or b.size[1] != x.size[1]:
            raise DimensionMismatch("apply: A %s, b %s, x %s" % (self.size, b.size, x.size))
        if b.vt != self.vt or x.vt != self.vt:
            raise NotSupported("mixed precision apply is not compiled (GINKGO_MIXED_PRECISION off)")

    def apply(self, *args):
        """apply(b, x) or apply(alpha, b, beta, x)"""
        if len(args) == 2:
            alpha = beta = None
            b, x = args
        elif len(args) == 4:
            alpha, b, beta, x = args
        else:
            raise TypeError("apply takes (b, x) or (alpha, b, beta, x)")
        self._check(b, x)
        e = self.exec
        with torch.cuda.stream(e.stream):
            bd = b.to_device(e)
            xd = x.to_device(e) if (alpha is not None or x.on_device) else Dense.create(
                e, x.size, dtype=x.values.dtype)
            ad = alpha.to_device(e) if alpha is not None else None
            btd = beta.to_device(e) if beta is not None else None
            self._apply_impl(ad, bd, btd, xd)
            if not x.on_device:
                x.values.copy_(xd.values, non_blocking=True)
                e.stream.synchronize()
        return x


class Csr(_SparseBase):
    """gko::matrix::Csr<ValueType, IndexType> on a B200Executor."""

    def __init__(self, exec_, size, values, col_idxs, row_ptrs):
        self.exec = exec_
        self.size = tuple(size)
        self.values, self.col_idxs, self.row_ptrs = values, col_idxs, row_ptrs
        self.nnz = values.numel()
        if row_ptrs.numel() != size[0] + 1:
            raise DimensionMismatch("row_ptrs must have num_rows + 1 entries")
        if values.dtype not in _VT or col_idxs.dtype not in _IT or row_ptrs.dtype != col_idxs.dtype:
            raise NotSupported("value/index type")
        self.vt, self.it = _VT[values.dtype], _IT[col_idxs.dtype]
        self._plan = None

    @staticmethod
    def create(exec_, size, values, col_idxs, row_ptrs):
        with torch.cuda.stream(exec_.stream):
            v, c, r = (t.to(exec_.device) for t in (values, col_idxs, row_ptrs))
        return Csr(exec_, size, v.contiguous(), c.contiguous(), r.contiguous())

    def plan(self):
        # the `srow` analogue: computed once per matrix (strategy->process in the reference)
        if self._plan is None:
            p = ctypes.c_void_p()
            fn = getattr(self.exec._l, "b200_csr_plan_create_%s_%s" % (self.vt, self.it))
            _lib.check(fn(self.exec.ctx, self.size[0], self.nnz, self.row_ptrs.data_ptr(),
                          ctypes.byref(p)))
            self._plan = p
            # this object owns the values tensor: callers that write into it call values_changed()
            self.exec._l.b200_csr_plan_allow_value_copy(p, 1)
            self.exec.run("b200_csr_plan_tune_%s_%s" % (self.vt, self.it), p, self.size[0],
                          self.size[1], self.nnz, self.row_ptrs, self.col_idxs, self.values)
        return self._plan

    def values_changed(self):
        """call after writing into .values in place: refreshes the plan's column-blocked value copy
        (b200_csr_plan_refresh_values_*; a no-op when the plan holds no copy)"""
        if self._plan is not None:
            self.exec.run("b200_csr_plan_refresh_values_%s_%s" % (self.vt, self.it), self._plan,
                          self.size[0], self.row_ptrs, self.values)

    def _apply_impl(self, alpha, b, beta, x):
        sfx = "_%s_%s" % (self.vt, self.it)
        common = (self.plan(), self.size[0], self.size[1], self.nnz, self.row_ptrs, self.col_idxs,
                  self.values)
        if alpha is None:
            self.exec.run("b200_csr_spmv" + sfx, *common, b.values, b.stride, b.size[1], x.values,
                          x.stride)
        else:
            self.exec.run("b200_csr_advanced_spmv" + sfx, *common, alpha.values, b.values, b.stride,
                          b.size[1], beta.values, x.values, x.stride)

    def __del__(self):
        try:
            if self._plan is not None:
                self.exec._l.b200_csr_plan_destroy(self._plan)
        except Exception:
            pass


# ---------------------------------------------------------------------------------------------
# Solvers: thin Python handles over the C++ host layer (ginkgo_b200/host/gko_b200.hpp) -- the
# loops, criteria and preconditioners run in C++; Python only passes device pointers.
# ---------------------------------------------------------------------------------------------
import os as _os

_HOST_LIB = None


def _configure_host_lib(h):
    """ctypes signatures of the gkob_* C handles (ginkgo_b200/host/capi.cpp)"""
    vp, ll, i, d = ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int, ctypes.c_double
    h.gkob_last_error.restype = ctypes.c_char_p
    h.gkob_exec_create.restype = vp
    h.gkob_exec_create.argtypes = [i, vp]
    h.gkob_destroy.argtypes = [vp]
    h.gkob_launch_count.restype = ll
    h.gkob_launch_count.argtypes = [vp]
    h.gkob_csr_kernel_variant.restype, h.gkob_csr_kernel_variant.argtypes = i, [vp]
    h.gkob_csr_plan_parts.restype, h.gkob_csr_plan_parts.argtypes = i, [vp]
    h.gkob_csr_gather_lines.restype, h.gkob_csr_gather_lines.argtypes = ctypes.c_double, [vp]
    h.gkob_staged_create.restype, h.gkob_staged_create.argtypes = vp, [vp, i, ll]
    h.gkob_staged_apply.restype, h.gkob_staged_apply.argtypes = i, [vp, vp, vp]
    h.gkob_staged_join.restype, h.gkob_staged_join.argtypes = i, [vp]
    h.gkob_staged_wait.restype, h.gkob_staged_wait.argtypes = i, [vp]
    h.gkob_staged_destroy.argtypes = [vp]
    h.gkob_csr_read_f64_i32.restype, h.gkob_csr_read_f64_i32.argtypes = vp, [vp, ctypes.c_char_p]
    h.gkob_csr_write_f64_i32.restype = i
    h.gkob_csr_write_f64_i32.argtypes = [vp, ctypes.c_char_p, i]
    h.gkob_read_f64_i32.restype, h.gkob_read_f64_i32.argtypes = vp, [vp, ctypes.c_char_p, ctypes.c_char_p]
    h.gkob_write_f64_i32.restype, h.gkob_write_f64_i32.argtypes = i, [vp, ctypes.c_char_p, i]
    h.gkob_num_rows.restype, h.gkob_num_rows.argtypes = ll, [vp]
    h.gkob_num_cols.restype, h.gkob_num_cols.argtypes = ll, [vp]
    h.gkob_solver_params.restype, h.gkob_solver_params.argtypes = None, [d, d, d]
    h.gkob_solver_guess.restype, h.gkob_solver_guess.argtypes = None, [i]
    h.gkob_solver_preconditioner.restype, h.gkob_solver_preconditioner.argtypes = None, [vp]
    h.gkob_csr_convert.restype = vp
    h.gkob_csr_convert.argtypes = [vp, ctypes.c_char_p, ll, ll, d, d]
    h.gkob_csr_sort_by_column_index.restype = i
    h.gkob_csr_sort_by_column_index.argtypes = [vp]
    h.gkob_csr_transpose.restype, h.gkob_csr_transpose.argtypes = vp, [vp]
    for s in ("f64", "f32"):
        for it in ("i32", "i64"):
            f = getattr(h, "gkob_csr_view_%s_%s" % (s, it))
            f.restype, f.argtypes = vp, [vp, ll, ll, ll, vp, vp, vp]
        f = getattr(h, "gkob_dense_view_" + s)
        f.restype, f.argtypes = vp, [vp, ll, ll, ll, vp]
        f = getattr(h, "gkob_solver_create_" + s)
        f.restype = vp
        f.argtypes = [vp, i, vp, i, vp, ll, ll, i, i, d, i, i, i, i, i]
        f = getattr(h, "gkob_solver_info_" + s)
        f.restype, f.argtypes = i, [vp, ctypes.POINTER(ll), ctypes.POINTER(ctypes.c_ubyte),
                                    ctypes.POINTER(i)]
        f = getattr(h, "gkob_solver_statuses_" + s)
        f.restype, f.argtypes = i, [vp, ctypes.POINTER(ctypes.c_ubyte), ll]
    h.gkob_jacobi_create.restype = vp
    h.gkob_jacobi_create.argtypes = [vp, i, vp, i, vp, ll, i, vp, ll, d]
    h.gkob_jacobi_get.restype, h.gkob_jacobi_get.argtypes = i, [vp, i, vp, vp, vp, vp, vp]
    h.gkob_jacobi_transpose.restype, h.gkob_jacobi_transpose.argtypes = vp, [vp]
    h.gkob_apply.restype, h.gkob_apply.argtypes = i, [vp, vp, vp]
    h.gkob_apply4.restype, h.gkob_apply4.argtypes = i, [vp, vp, vp, vp, vp]
    h.gkob_synchronize.restype, h.gkob_synchronize.argtypes = i, [vp]
    # distributed set-up
    h.gkob_partition_from_mapping.restype, h.gkob_partition_from_mapping.argtypes = vp, [vp, vp, ll, i]
    h.gkob_partition_from_contiguous.restype = vp
    h.gkob_partition_from_contiguous.argtypes = [vp, vp, ll, vp]
    h.gkob_partition_uniform.restype, h.gkob_partition_uniform.argtypes = vp, [vp, i, ll]
    h.gkob_partition_info.restype, h.gkob_partition_info.argtypes = i, [vp, vp, vp, vp, vp, vp]
    h.gkob_partition_destroy.restype, h.gkob_partition_destroy.argtypes = None, [vp]
    h.gkob_dist_assemble_f64_i32.restype = vp
    h.gkob_dist_assemble_f64_i32.argtypes = [vp, vp, vp, i, ll, ll, ll, vp, vp, vp]
    h.gkob_dist_assembly_sizes.restype, h.gkob_dist_assembly_sizes.argtypes = i, [vp, vp]
    h.gkob_dist_assembly_get.restype, h.gkob_dist_assembly_get.argtypes = i, [vp, vp, vp, vp, vp, vp, vp]
    h.gkob_dist_assembly_map_to_local.restype = i
    h.gkob_dist_assembly_map_to_local.argtypes = [vp, i, ll, vp, vp]
    h.gkob_dist_assembly_destroy.restype, h.gkob_dist_assembly_destroy.argtypes = None, [vp]
    h.gkob_dist_send_layout.restype, h.gkob_dist_send_layout.argtypes = i, [i, i, vp, vp, vp]
    h.gkob_dist_matrix_read_f64_i32.restype = vp
    h.gkob_dist_matrix_read_f64_i32.argtypes = [vp, vp, i, i, vp, ll, ll, ll, vp, vp, vp, i]
    h.gkob_dist_matrix_sizes.restype, h.gkob_dist_matrix_sizes.argtypes = i, [vp, vp, vp]
    return h


def _host():
    global _HOST_LIB
    if _HOST_LIB is None:
        _lib.lib()  # the C-ABI library first (RTLD_GLOBAL)
        path = _os.path.join(_os.path.dirname(_os.path.abspath(__file__)), "lib",
                             "libgko_b200_host.so")
        if not _os.path.exists(path):
            raise _lib.B200Error("%s not found: run `make -C ginkgo_b200/host`" % path)
        _HOST_LIB = _configure_host_lib(ctypes.CDLL(path))
    return _HOST_LIB


def _hcheck(rc):
    if rc != 0:
        msg = _host().gkob_last_error().decode()
        if rc == 2:
            raise DimensionMismatch(msg)
        if rc == 3:
            raise NotSupported(msg)
        raise _lib.B200Error(msg)


class HostExecutor:
    """gko_b200::B200Executor (C++) bound to a torch stream"""

    def __init__(self, device_id=0, stream=None):
        self.device = torch.device("cuda", device_id)
        with torch.cuda.device(device_id):
            self.stream = stream or torch.cuda.Stream(device_id)
        self.h = _host().gkob_exec_create(device_id, self.stream.cuda_stream)
        if not self.h:
            raise _lib.B200Error(_host().gkob_last_error().decode())

    def synchronize(self):
        _hcheck(_host().gkob_synchronize(self.h))

    def launch_count(self):
        return _host().gkob_launch_count(self.h)


class _HostObj:
    def __init__(self, exec_, handle, keep=()):
        if not handle:
            raise _lib.B200Error(_host().gkob_last_error().decode())
        self.exec, self.h, self._keep = exec_, handle, keep
        self._hl = _host()  # destroyed by the library that made it (tests swap in a host-memory mock)

    def __del__(self):
        try:
            self._hl.gkob_destroy(self.h)
        except Exception:
            pass


def host_csr(exec_, size, values, col_idxs, row_ptrs):
    """gko_b200::matrix::Csr<V,int32> (int64 index tensors: Csr<V,int64>) viewing torch device tensors"""
    s = _VT[values.dtype]
    fn = getattr(_host(), "gkob_csr_view_%s_%s" % (s, "i64" if col_idxs.dtype == torch.int64 else "i32"))
    o = _HostObj(exec_, fn(exec_.h, size[0], size[1], values.numel(), row_ptrs.data_ptr(),
                           col_idxs.data_ptr(), values.data_ptr()), (values, col_idxs, row_ptrs))
    o.vt = s
    return o


_HYB = {"automatic": 0, "column_limit": 1, "imbalance_limit": 2, "imbalance_bounded_limit": 3,
        "minimal_storage_limit": 4}


def host_convert(A, fmt, slice_size=64, stride_factor=1, strategy="automatic", columns=0,
                 percent=0.8, ratio=0.0001):
    """Csr::convert_to(Ell | Sellp | Coo | Hybrid) on the device; returns the new LinOp"""
    p0, p1 = (slice_size, stride_factor) if fmt == "sellp" else (_HYB[strategy], columns)
    o = _HostObj(A.exec, _host().gkob_csr_convert(A.h, fmt.encode(), p0, p1, float(percent),
                                                  float(ratio)))
    o.vt = A.vt
    return o


def host_sort_by_column_index(A):
    """Csr::sort_by_column_index in place (on the tensors the handle views)"""
    _hcheck(_host().gkob_csr_sort_by_column_index(A.h))


def host_transpose(A):
    """Transposable::transpose of a Csr handle -> a new (owning) handle"""
    t = _HostObj(A.exec, _host().gkob_csr_transpose(A.h), keep=(A,))
    t.vt = getattr(A, "vt", None)
    return t


AUTODETECT = 0xff  # gko::precision_reduction::autodetect()


def precision_reduction(preserving, nonpreserving):
    """the byte of gko::precision_reduction(preserving, nonpreserving)"""
    return (preserving << 4) | nonpreserving


def host_jacobi(A, max_block_size, block_ptrs=None, storage_optimization=None, accuracy=0.1):
    """gko_b200::preconditioner::Jacobi<V,int32>::build().with_max_block_size(..)
    [.with_block_pointers(..)] [.with_storage_optimization(..)] [.with_accuracy(..)].on(exec)->generate(A).
    storage_optimization: None | one precision_reduction byte (AUTODETECT = 0xff) | a sequence of bytes
    (block-wise, replicated cyclically).  Returns a LinOp handle (host_apply / host_jacobi_get)."""
    import numpy as _np
    bp = None if block_ptrs is None else _np.ascontiguousarray(block_ptrs, dtype=_np.int32)
    if storage_optimization is None:
        kind, so = 0, _np.zeros(1, _np.uint8)
    elif _np.isscalar(storage_optimization):
        kind, so = 1, _np.array([storage_optimization], _np.uint8)
    else:
        kind, so = 2, _np.ascontiguousarray(storage_optimization, dtype=_np.uint8)
    o = _HostObj(A.exec, _host().gkob_jacobi_create(
        A.exec.h, 0 if A.vt == "f64" else 1, A.h, int(max_block_size),
        None if bp is None else bp.ctypes.data, 0 if bp is None else len(bp) - 1, kind, so.ctypes.data, len(so),
        float(accuracy)), keep=(A,))
    o.vt = A.vt
    return o


def host_jacobi_get(J):
    """storage scheme, raw block storage (as the value type), block pointers, the precision_reduction
    byte of every block (None without storage optimisation) and the condition numbers, on the host"""
    import numpy as _np
    vt = 0 if J.vt == "f64" else 1
    dt = _np.float64 if vt == 0 else _np.float32
    meta = _np.zeros(6, _np.int64)
    _hcheck(_host().gkob_jacobi_get(J.h, vt, meta.ctypes.data, None, None, None, None))
    nb, stored = int(meta[3]), int(meta[4])
    blocks = _np.zeros(max(stored, 1), dt)
    ptrs = _np.zeros(nb + 1, _np.int32)
    prec = _np.zeros(max(nb, 1), _np.uint8)
    cond = _np.zeros(max(nb, 1), dt)
    J.exec.synchronize()
    _hcheck(_host().gkob_jacobi_get(J.h, vt, meta.ctypes.data, blocks.ctypes.data, ptrs.ctypes.data,
                                    prec.ctypes.data, cond.ctypes.data))
    return dict(block_offset=int(meta[0]), group_offset=int(meta[1]), group_power=int(meta[2]), num_blocks=nb,
                blocks=blocks[:stored], block_ptrs=ptrs, precisions=prec[:nb] if meta[5] else None,
                conditioning=cond[:nb] if meta[5] else None)


def host_jacobi_transpose(J):
    """Jacobi::transpose()"""
    t = _HostObj(J.exec, _host().gkob_jacobi_transpose(J.h), keep=(J,))
    t.vt = J.vt
    return t


def host_apply(op, b, x, alpha=None, beta=None):
    """x = op(b)  or  x = alpha op(b) + beta x   (handles of host_dense; alpha / beta 1x1)"""
    if alpha is None:
        _hcheck(_host().gkob_apply(op.h, b.h, x.h))
    else:
        _hcheck(_host().gkob_apply4(op.h, alpha.h, b.h, beta.h, x.h))


class StagedApply:
    """gko_b200::staged_apply<V>: x_host = op(b_host) with HOST tensors (pinned to overlap),
    pipelined over two copy streams; apply() is asynchronous, wait() makes x_host valid."""

    def __init__(self, A, nrhs=1):
        self.A = A
        self._hl = _host()
        self.h = self._hl.gkob_staged_create(A.h, 0 if A.vt == "f64" else 1, nrhs)
        if not self.h:
            raise _lib.B200Error(_host().gkob_last_error().decode())

    def apply(self, b_host, x_host):
        assert not b_host.is_cuda and not x_host.is_cuda
        _hcheck(_host().gkob_staged_apply(self.h, b_host.data_ptr(), x_host.data_ptr()))

    def join(self):
        _hcheck(_host().gkob_staged_join(self.h))

    def wait(self):
        _hcheck(_host().gkob_staged_wait(self.h))

    def __del__(self):
        try:
            self._hl.gkob_staged_destroy(self.h)
        except Exception:
            pass


def host_read_csr(exec_, path):
    """gko::read_generic<Csr<double,int32>>: MatrixMarket or Ginkgo-binary file -> device Csr"""
    o = _HostObj(exec_, _host().gkob_csr_read_f64_i32(exec_.h, str(path).encode()))
    o.vt = "f64"
    o.size = (_host().gkob_num_rows(o.h), _host().gkob_num_cols(o.h))
    return o


def host_write_csr(A, path, layout="coordinate"):
    """gko::write / gko::write_binary of a device Csr<double,int32>"""
    _hcheck(_host().gkob_csr_write_f64_i32(A.h, str(path).encode(),
                                           {"coordinate": 0, "array": 1, "binary": 2}[layout]))


def host_read(exec_, path, fmt="csr"):
    """gko::read_generic<Format<double,int32>>: fmt csr | ell | sellp | coo | hybrid"""
    o = _HostObj(exec_, _host().gkob_read_f64_i32(exec_.h, str(path).encode(), fmt.encode()))
    o.vt = "f64"
    o.size = (_host().gkob_num_rows(o.h), _host().gkob_num_cols(o.h))
    return o


def host_write(A, path, layout="coordinate"):
    """gko::write / gko::write_binary of any of the five formats (double, int32)"""
    _hcheck(_host().gkob_write_f64_i32(A.h, str(path).encode(), {"coordinate": 0, "array": 1, "binary": 2}[layout]))


def host_dense(exec_, t, cols=None, stride=None):
    """gko_b200::matrix::Dense<V> viewing a torch device tensor (rows x stride, row-major)"""
    if t.dim() == 1:
        t = t.reshape(-1, 1)
    rows, st = t.shape[0], (stride or t.shape[1])
    cols = cols or t.shape[1]
    fn = getattr(_host(), "gkob_dense_view_" + _VT[t.dtype])
    return _HostObj(exec_, fn(exec_.h, rows, cols, st, t.data_ptr()), (t,))


class HostSolver:
    """solver::Cg / Bicgstab / Gmres of the C++ host layer.

    kind: "cg" | "bicgstab" | "gmres" | "fcg" | "cgs" | "pipe_cg" | "gcr" (krylov_dim) | "minres" | "bicg" | "ir" (relaxation_factor) | "chebyshev" (foci);  criteria: max_iters (None = no Iteration criterion),
    res_kind 0 none / 1 ResidualNorm / 2 ImplicitResidualNorm, baseline 0 rhs_norm /
    1 initial_resnorm / 2 absolute, iter_first = order inside stop::Combined;
    precond_max_bs 0 = none, 1 = scalar Jacobi, k > 1 = block Jacobi (block_ptrs given, or
    detected by find_blocks); for "ir" the preconditioner slot is the inner solver.
    fused: Cg's device-resident iteration (on where applicable); fused_multi_rhs: Cg's device-resident
    iteration for 2..32 right-hand sides, opt-in (Csr, b and x without gaps between columns, Identity or
    scalar Jacobi, Iteration / (Implicit)ResidualNorm; one matrix pass per iteration for all columns,
    each column stops on its own); fused_bicgstab: Bicgstab's, opt-in; fused_bicgstab_multi_rhs:
    Bicgstab's for 2..32 right-hand sides, opt-in, with fused_multi_rhs's admission (one matrix pass per
    SpMV for all columns; each column stops on its own, at the top or the mid-iteration check);
    fused_gmres: Gmres's, opt-in (modified Gram-Schmidt, one right-hand side, Identity or any Jacobi,
    Iteration / ResidualNorm criteria; anything else takes the loop); fused_gmres_multi_rhs: Gmres's
    for 2..32 right-hand sides, opt-in and independent of fused_gmres (MGS, CGS or CGS2, b and x without
    gaps between columns, Identity or scalar Jacobi, Iteration / ResidualNorm; one matrix pass per SpMV
    for all columns, each column stops on its own; block Jacobi and anything else take the loop);
    fused_minres: Minres's, opt-in (Csr, one right-hand side, Identity or scalar Jacobi, Iteration /
    ImplicitResidualNorm; three launches per iteration; ResidualNorm and anything else take the loop);
    fused_minres_multi_rhs: Minres's for 2..32 right-hand sides, opt-in and independent of fused_minres
    (b and x without gaps between columns, otherwise fused_minres's admission; one matrix pass per
    iteration for all columns, each column stops on its own).
    check_every: iterations per graph launch on those paths.  preconditioner: a generated one (host_jacobi, e.g. with
    storage_optimization) used in place of precond_max_bs.  used_fused tells after apply whether such a
    path ran; stop_status is column 0's stopping status, stop_statuses every column's."""

    def __init__(self, exec_, kind, A, precond_max_bs=0, block_ptrs=None, max_iters=None,
                 res_kind=1, baseline=0, reduction=1e-8, iter_first=True, krylov_dim=30, ortho=0,
                 fused=True, check_every=16, relaxation_factor=1.0, foci=(0.0, 1.0), initial_guess="provided",
                 fused_bicgstab=False, fused_gmres=False, preconditioner=None, fused_multi_rhs=False,
                 fused_bicgstab_multi_rhs=False, fused_gmres_multi_rhs=False, fused_minres=False,
                 fused_minres_multi_rhs=False):
        self.vt = A.vt
        _host().gkob_solver_params(float(relaxation_factor), float(foci[0]), float(foci[1]))
        # "ir" only: solver::initial_guess_mode of with_default_initial_guess
        _host().gkob_solver_guess({"provided": 0, "zero": 1, "rhs": 2}[initial_guess])
        # a generated preconditioner (host_jacobi) instead of precond_max_bs / block_ptrs
        _host().gkob_solver_preconditioner(None if preconditioner is None else preconditioner.h)
        bp = None
        nb = 0
        if block_ptrs is not None:
            import numpy as np
            self._bp = np.ascontiguousarray(block_ptrs, dtype=np.int32)
            bp, nb = self._bp.ctypes.data, len(self._bp) - 1
        fn = getattr(_host(), "gkob_solver_create_" + self.vt)
        self.obj = _HostObj(exec_, fn(exec_.h, {"cg": 0, "bicgstab": 1, "gmres": 2, "fcg": 3, "cgs": 4, "ir": 5, "chebyshev": 6, "pipe_cg": 7, "gcr": 8, "minres": 9, "bicg": 10}[kind], A.h,
                                      precond_max_bs, bp, nb, -1 if max_iters is None else max_iters,
                                      res_kind, baseline, reduction, int(iter_first), krylov_dim,
                                      ortho, int(bool(fused)) | (2 if fused_bicgstab else 0) |
                                      (4 if fused_gmres else 0) | (8 if fused_multi_rhs else 0) |
                                      (16 if fused_bicgstab_multi_rhs else 0) |
                                      (32 if fused_gmres_multi_rhs else 0) |
                                      (64 if fused_minres else 0) |
                                      (128 if fused_minres_multi_rhs else 0),
                                      check_every), (A,))

    def apply(self, b, x):
        _hcheck(_host().gkob_apply(self.obj.h, b.h, x.h))
        it, st, fu = ctypes.c_longlong(0), ctypes.c_ubyte(0), ctypes.c_int(0)
        _hcheck(getattr(_host(), "gkob_solver_info_" + self.vt)(self.obj.h, ctypes.byref(it),
                                                                ctypes.byref(st), ctypes.byref(fu)))
        self.num_iterations, self.stop_status, self.used_fused = it.value, st.value, bool(fu.value)
        cols = _host().gkob_num_cols(b.h)
        sts = (ctypes.c_ubyte * max(cols, 1))()
        _hcheck(getattr(_host(), "gkob_solver_statuses_" + self.vt)(self.obj.h, sts, cols))
        self.stop_statuses = list(sts[:cols])
        return x


# ---------------------------------------------------------------------------------------------
# Multi-GPU: row-partitioned Csr + fused distributed CG (C++: host/gko_b200_dist.hpp)
# ---------------------------------------------------------------------------------------------
def _np(a, dtype):
    import numpy as np
    return np.ascontiguousarray(a, dtype)


class HostPartition:
    """gko_b200::distributed::Partition<int32, int64> (experimental::distributed::Partition):
    built on the device from host descriptions"""

    def __init__(self, exec_, handle):
        if not handle:
            raise _lib.B200Error(_host().gkob_last_error().decode())
        self.exec, self.h, self._hl = exec_, handle, _host()

    @classmethod
    def from_mapping(cls, exec_, mapping, num_parts):
        m = _np(mapping, "int32")
        return cls(exec_, _host().gkob_partition_from_mapping(exec_.h, m.ctypes.data, len(m), num_parts))

    @classmethod
    def from_contiguous(cls, exec_, ranges, part_ids=None):
        r = _np(ranges, "int64")
        ids = None if part_ids is None else _np(part_ids, "int32")
        if len(r) == 0 or (ids is not None and len(ids) != len(r) - 1):
            raise DimensionMismatch("Partition: ranges needs num_ranges + 1 entries, part_ids num_ranges")
        return cls(exec_, _host().gkob_partition_from_contiguous(
            exec_.h, r.ctypes.data, len(r) - 1, None if ids is None else ids.ctypes.data))

    @classmethod
    def uniform(cls, exec_, num_parts, global_size):
        return cls(exec_, _host().gkob_partition_uniform(exec_.h, num_parts, global_size))

    def info(self):
        import numpy as np
        meta = np.zeros(6, np.int64)
        _hcheck(_host().gkob_partition_info(self.h, meta.ctypes.data, None, None, None, None))
        nr, npart = int(meta[1]), int(meta[2])
        bounds = np.zeros(nr + 1, np.int64)
        ids, start = np.zeros(max(nr, 1), np.int32), np.zeros(max(nr, 1), np.int32)
        sizes = np.zeros(max(npart, 1), np.int32)
        _hcheck(_host().gkob_partition_info(self.h, meta.ctypes.data, bounds.ctypes.data, ids.ctypes.data,
                                            start.ctypes.data, sizes.ctypes.data))
        return dict(size=int(meta[0]), num_ranges=nr, num_parts=npart, num_empty_parts=int(meta[3]),
                    connected=bool(meta[4]), ordered=bool(meta[5]), range_bounds=bounds, part_ids=ids[:nr],
                    starting_indices=start[:nr], part_sizes=sizes[:npart])

    def __del__(self):
        try:
            self._hl.gkob_partition_destroy(self.h)
        except Exception:
            pass


class HostAssembly:
    """gko_b200::distributed::assemble_local<double, int32, int64>: what part `rank` owns of the
    global (row-major sorted) triplets, columns in the combined index space"""

    def __init__(self, exec_, row_part, rank, shape, rows, cols, vals, col_part=None):
        import numpy as np
        r, c, v = _np(rows, "int64"), _np(cols, "int64"), _np(vals, "float64")
        self._hl = _host()
        self.h = self._hl.gkob_dist_assemble_f64_i32(
            exec_.h, row_part.h, None if col_part is None else col_part.h, rank, shape[0], shape[1], len(r),
            r.ctypes.data, c.ctypes.data, v.ctypes.data)
        if not self.h:
            msg = _host().gkob_last_error().decode()
            raise (DimensionMismatch if msg.startswith("DimensionMismatch") else _lib.B200Error)(msg)
        sz = np.zeros(5, np.int64)
        _hcheck(_host().gkob_dist_assembly_sizes(self.h, sz.ctypes.data))
        self.n_local_rows, self.n_local_cols, self.n_ghost, self.nnz, nparts = (int(x) for x in sz)
        self.row_ptrs = np.zeros(self.n_local_rows + 1, np.int32)
        self.col_idxs = np.zeros(max(self.nnz, 1), np.int32)
        self.values = np.zeros(max(self.nnz, 1))
        self.recv_counts = np.zeros(max(nparts, 1), np.int64)
        self.remote_global = np.zeros(max(self.n_ghost, 1), np.int64)
        self.remote_local = np.zeros(max(self.n_ghost, 1), np.int32)
        _hcheck(_host().gkob_dist_assembly_get(self.h, self.row_ptrs.ctypes.data, self.col_idxs.ctypes.data,
                                               self.values.ctypes.data, self.recv_counts.ctypes.data,
                                               self.remote_global.ctypes.data, self.remote_local.ctypes.data))
        self.col_idxs, self.values = self.col_idxs[:self.nnz], self.values[:self.nnz]
        self.recv_counts = self.recv_counts[:nparts]
        self.remote_global, self.remote_local = self.remote_global[:self.n_ghost], self.remote_local[:self.n_ghost]

    def map_to_local(self, global_ids, index_space):
        import numpy as np
        g = _np(global_ids, "int64")
        out = np.zeros(max(len(g), 1), np.int32)
        _hcheck(_host().gkob_dist_assembly_map_to_local(self.h, index_space, len(g), g.ctypes.data,
                                                        out.ctypes.data))
        return out[:len(g)]

    def __del__(self):
        try:
            self._hl.gkob_dist_assembly_destroy(self.h)
        except Exception:
            pass


def host_send_layout(num_parts, rank, S):
    """S[q][p] = entries rank q receives from p -> (send_counts, source_offsets) of `rank`"""
    import numpy as np
    S = _np(S, "int64")
    sc, so = np.zeros(num_parts, np.int64), np.zeros(num_parts, np.int64)
    _hcheck(_host().gkob_dist_send_layout(num_parts, rank, S.ctypes.data, sc.ctypes.data, so.ctypes.data))
    return sc, so


class DistMatrix:
    """experimental::distributed::Matrix analogue.  Each rank passes ITS rows (row_ptrs local,
    col_idxs GLOBAL, values) and the partition offsets; set-up uses torch.distributed
    (ginkgo_b200/distributed.py), the per-apply halo exchange uses the library's own NCCL
    communicator on the executor's stream."""

    @staticmethod
    def _bind(h):
        vp, ll, i = ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int
        h.gkob_dist_unique_id.restype, h.gkob_dist_unique_id.argtypes = i, [vp]
        h.gkob_dist_matrix_create_f64_i32.restype = vp
        h.gkob_dist_matrix_create_f64_i32.argtypes = [vp, vp, i, i, ll, ll, ll, vp, vp, vp, vp, vp, vp]
        h.gkob_dist_spmv_f64.restype, h.gkob_dist_spmv_f64.argtypes = i, [vp, vp, vp]
        h.gkob_dist_last_ghosts_f64.restype, h.gkob_dist_last_ghosts_f64.argtypes = i, [vp, vp]
        h.gkob_dist_set_overlap.restype, h.gkob_dist_set_overlap.argtypes = i, [vp, i]
        h.gkob_dist_pipelined.restype, h.gkob_dist_pipelined.argtypes = i, [vp]
        h.gkob_dist_p2p.restype, h.gkob_dist_p2p.argtypes = i, [vp]
        h.gkob_dist_cg_create_f64.restype = i
        h.gkob_dist_cg_create_f64.argtypes = [vp, i, ll, i, i, ctypes.c_double, i, i]
        h.gkob_dist_cg_apply_f64.restype = i
        h.gkob_dist_cg_apply_f64.argtypes = [vp, vp, vp, ctypes.POINTER(ll),
                                             ctypes.POINTER(ctypes.c_ubyte)]
        h.gkob_dist_destroy.argtypes = [vp]
        h.gkob_dist_vector_read_f64.restype = i
        h.gkob_dist_vector_read_f64.argtypes = [vp, vp, ll, ll, ll, vp, vp, vp, vp]
        h.gkob_dist_solve_f64.restype = i
        h.gkob_dist_solve_f64.argtypes = [vp, i, i, i, vp, vp, ll, ll, i, i, ctypes.c_double, i, i, i, i,
                                          ctypes.POINTER(ll), ctypes.POINTER(ctypes.c_ubyte)]
        h.gkob_dist_apply_f64.restype, h.gkob_dist_apply_f64.argtypes = i, [vp, vp, vp, i]

    @staticmethod
    def _unique_id(exec_, rank, world, group):
        """NCCL unique id from rank 0, broadcast over torch.distributed"""
        import torch.distributed as dist
        h = _host()
        idt = torch.zeros(128, dtype=torch.uint8)
        if rank == 0:
            buf = (ctypes.c_ubyte * 128)()
            _hcheck(h.gkob_dist_unique_id(buf))
            idt = torch.tensor(list(buf), dtype=torch.uint8)
        if world > 1:
            idt = idt.to(exec_.device)
            dist.broadcast(idt, 0, group=group)
            idt = idt.cpu()
        return (ctypes.c_ubyte * 128)(*idt.tolist())

    def __init__(self, exec_, offsets, row_ptrs, col_idxs_global, values, group=None):
        import torch.distributed as dist
        from . import distributed as D
        h = _host()
        self._bind(h)
        self.exec = exec_
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        with torch.cuda.stream(exec_.stream):
            part = D.build_partition(col_idxs_global, offsets, self.rank, group)
            exec_.stream.synchronize()
        self.part = part
        self.n_local, self.n_ghost = part["n_local"], part["n_ghost"]
        self.row_ptrs, self.values = row_ptrs, values
        self.col_idxs = part["col_idxs_local"].contiguous()
        self.send_idx = part["send_idx"].contiguous()
        idb = self._unique_id(exec_, self.rank, self.world, group)
        sc = (ctypes.c_longlong * self.world)(*part["send_counts"].tolist())
        rc = (ctypes.c_longlong * self.world)(*part["recv_counts"].tolist())
        self._hl = h
        self.h = h.gkob_dist_matrix_create_f64_i32(
            exec_.h, idb, self.rank, self.world, self.n_local, self.n_ghost, values.numel(),
            row_ptrs.data_ptr(), self.col_idxs.data_ptr(), values.data_ptr(), sc, rc,
            self.send_idx.data_ptr() if self.send_idx.numel() else None)
        if not self.h:
            raise _lib.B200Error(h.gkob_last_error().decode())

    @classmethod
    def read(cls, exec_, partition, shape, rows, cols, vals, group=None, keep_local_block=False):
        """experimental::distributed::Matrix::read_distributed: every rank passes the global
        (row-major sorted) triplets -- or at least its own rows -- and a HostPartition with one
        part per rank; the split, the column renumbering and the exchange of the send lists run
        in the library (device kernels + its own communicator).  keep_local_block: also keep the
        square block of the owned columns (needed by solve(..., schwarz != 0)).  Collective."""
        import torch.distributed as dist
        h = _host()
        cls._bind(h)
        self = cls.__new__(cls)
        self.exec = exec_
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        idb = cls._unique_id(exec_, self.rank, self.world, group)
        r, c, v = _np(rows, "int64"), _np(cols, "int64"), _np(vals, "float64")
        self._hl = h
        self.h = h.gkob_dist_matrix_read_f64_i32(exec_.h, idb, self.rank, self.world, partition.h, shape[0],
                                                 shape[1], len(r), r.ctypes.data, c.ctypes.data, v.ctypes.data,
                                                 int(keep_local_block))
        if not self.h:
            raise _lib.B200Error(h.gkob_last_error().decode())
        import numpy as np
        sz = np.zeros(3, np.int64)
        _hcheck(h.gkob_dist_matrix_sizes(self.h, sz.ctypes.data, None))
        self.n_local, self.n_local_cols, self.n_ghost = (int(x) for x in sz)
        self.ghost_globals = np.zeros(max(self.n_ghost, 1), np.int64)
        _hcheck(h.gkob_dist_matrix_sizes(self.h, sz.ctypes.data, self.ghost_globals.ctypes.data))
        self.ghost_globals = self.ghost_globals[:self.n_ghost]
        return self

    @property
    def p2p(self):
        """bit 0: scalar all-reduces on peer memory, bit 1: halo exchange on peer memory"""
        return _host().gkob_dist_p2p(self.h)

    def apply(self, x_ext, y_local):
        """y_local = A x; x_ext is [n_local owned | n_ghost].  The ghosts are exchanged; on the
        peer-memory path the SpMV reads them in place from the landing slot (last_ghosts() returns
        them), otherwise they are written into the tail of x_ext"""
        _hcheck(_host().gkob_dist_spmv_f64(self.h, x_ext.data_ptr(), y_local.data_ptr()))

    def set_overlap(self, on):
        """opt into the pipelined exchange: owner blocks applied in arrival order while the rest of x is
        still in flight (row sums re-associated: 1e-13-equal, not bit-equal, to one GPU)"""
        _hcheck(_host().gkob_dist_set_overlap(self.h, int(bool(on))))

    @property
    def pipelined(self):
        return bool(_host().gkob_dist_pipelined(self.h))

    def last_ghosts(self):
        """the ghost values the last apply() gathered from (device tensor of n_ghost entries)"""
        out = torch.empty(max(self.n_ghost, 1), dtype=torch.float64, device=self.exec.device)
        _hcheck(_host().gkob_dist_last_ghosts_f64(self.h, out.data_ptr()))
        return out[:self.n_ghost]

    def solve(self, kind, b_local, x_local, global_rows, precond_max_bs=0, max_iters=None, res_kind=1,
              baseline=0, reduction=1e-8, iter_first=True, krylov_dim=30, ortho=0, schwarz=0):
        """any host-layer solver (HostSolver's kinds) on the distributed matrix: b_local / x_local are
        this rank's rows, wrapped as distributed::Vector (dots and norms sum over the ranks); the
        preconditioner is Jacobi(precond_max_bs) generated from the local block (schwarz=0), or
        distributed::preconditioner::Schwarz around that Jacobi on the square local block (schwarz=-1)
        or around `schwarz` Richardson sweeps preconditioned by it.  Collective.  -> (iterations, status)"""
        kinds = {"cg": 0, "bicgstab": 1, "gmres": 2, "fcg": 3, "cgs": 4, "ir": 5, "chebyshev": 6, "pipe_cg": 7,
                 "gcr": 8, "minres": 9, "bicg": 10}
        it, st = ctypes.c_longlong(0), ctypes.c_ubyte(0)
        _hcheck(_host().gkob_dist_solve_f64(
            self.h, kinds[kind], precond_max_bs, schwarz, b_local.data_ptr(), x_local.data_ptr(), global_rows,
            -1 if max_iters is None else max_iters, res_kind, baseline, reduction, int(iter_first), krylov_dim,
            ortho, 1 if b_local.dim() == 1 else b_local.shape[1], ctypes.byref(it), ctypes.byref(st)))
        return it.value, st.value

    def apply_local(self, b_local, x_local):
        """LinOp::apply on the local rows of distributed vectors (n_local [x nrhs] tensors): the owned
        entries are copied next to the ghost slots of an internal extended vector"""
        _hcheck(_host().gkob_dist_apply_f64(self.h, b_local.data_ptr(), x_local.data_ptr(),
                                            1 if b_local.dim() == 1 else b_local.shape[1]))

    def make_cg(self, scalar_jacobi=False, max_iters=None, res_kind=1, baseline=0, reduction=1e-8,
                iter_first=True, check_every=16):
        _hcheck(_host().gkob_dist_cg_create_f64(self.h, int(scalar_jacobi),
                                                -1 if max_iters is None else max_iters, res_kind,
                                                baseline, reduction, int(iter_first), check_every))

    def cg_apply(self, b_local, x_local):
        it, st = ctypes.c_longlong(0), ctypes.c_ubyte(0)
        _hcheck(_host().gkob_dist_cg_apply_f64(self.h, b_local.data_ptr(), x_local.data_ptr(),
                                               ctypes.byref(it), ctypes.byref(st)))
        return it.value, st.value

    def __del__(self):
        try:
            self._hl.gkob_dist_destroy(self.h)
        except Exception:
            pass
