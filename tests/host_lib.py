"""ctypes binding of implicit-sdf-planner_b200/host/libisdf_host.so (the C++ host adapters' test hooks)."""
import ctypes as C
import os
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "implicit-sdf-planner_b200", "host", "libisdf_host.so")
dp = C.POINTER(C.c_double)
_lib = None


def lib():
    global _lib
    if _lib is None:
        import isdf_b200 as I
        I.load_library()   # libisdf_b200.so first (rpath also finds it)
        L = C.CDLL(LIB)
        L.isdf_host_minco_forward.argtypes = [C.c_int, dp, dp, dp, dp, dp, dp, dp, dp]
        L.isdf_host_minco_backward.argtypes = [C.c_int, dp, dp, dp, dp, dp, dp, dp, dp]
        L.isdf_host_backend_create.restype = C.c_void_p
        L.isdf_host_backend_create.argtypes = [C.c_void_p, C.c_int, dp, dp, C.c_double, C.c_int, C.c_int]
        L.isdf_host_backend_cost.restype = C.c_double
        L.isdf_host_backend_cost.argtypes = [C.c_void_p, dp, dp, C.c_int]
        L.isdf_host_backend_last.argtypes = [C.c_void_p, dp, dp, dp, C.POINTER(C.c_int)]
        L.isdf_host_backend_destroy.argtypes = [C.c_void_p]
        L.isdf_host_tau_maps.argtypes = [dp, C.c_int, dp, dp]
        L.isdf_host_shape_sdf_grad.restype = C.c_double
        L.isdf_host_shape_sdf_grad.argtypes = [C.c_void_p, dp, dp]
        L.isdf_host_lbfgs_generic_ex.argtypes = [C.c_int, dp, dp, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int,
                                                 C.c_int] + [C.c_double] * 5 + [C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.isdf_host_lbfgs_backend.argtypes = [C.c_void_p, dp, C.c_int, dp, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int,
                                              C.POINTER(C.c_int), C.POINTER(C.c_int)]
        ip = C.POINTER(C.c_int)
        L.isdf_host_read_obj.argtypes = [C.c_char_p, dp, C.c_int, C.POINTER(C.c_int32), C.c_int, ip, ip]
        L.isdf_host_set_shape_obj.argtypes = [C.c_void_p, C.c_char_p, dp]
        L.isdf_host_lbfgs_batch_generic_ex.argtypes = [C.c_int, C.c_int, dp, dp, ip, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double,
                                                       C.c_int, C.c_int] + [C.c_double] * 5 + [C.c_int, ip, ip]
        L.isdf_host_lbfgs_batch_backend.argtypes = [C.c_void_p, C.c_int, C.c_int, dp, dp, C.c_double, dp, dp, ip, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int,
                                                    ip, ip, ip]
        _lib = L
    return _lib


EVAL_T = C.CFUNCTYPE(C.c_double, C.c_void_p, dp, dp, C.c_int, dp)   # lbfgs_eval_raw_t


# lbfgs_parameter_t's defaults (lbfgs.hpp:40-142) but min_step, which is config_CappedCone.yaml:101's
LS_DEFAULTS = dict(max_linesearch=64, min_step=1e-32, max_step=1e20, f_dec_coeff=1e-4, cautious_factor=1e-6, machine_prec=1e-16)


def _ls_args(max_linesearch, min_step, max_step, f_dec_coeff, cautious_factor, machine_prec):
    return [int(max_linesearch), float(min_step), float(max_step), float(f_dec_coeff), float(cautious_factor), float(machine_prec)]


def lbfgs_minimize(fun, x0, mem_size=8, past=3, delta=1e-6, g_epsilon=1e-5, max_iterations=0, **ls):
    """fun(x) -> (f, grad). Runs the product's L-BFGS driver on a python callback (KATs, CPU baseline). ls: any of LS_DEFAULTS' keys."""
    x = f(x0).copy()
    n = x.size
    count = [0]

    trace = []

    def cb(_inst, xp, gp, nn, pc):
        xv = np.ctypeslib.as_array(xp, shape=(nn,))
        trace.append(xv.copy())
        fv, gv = fun(xv.copy())
        np.ctypeslib.as_array(gp, shape=(nn,))[:] = gv
        count[0] += 1
        return float(fv)
    cfn = EVAL_T(cb)
    fx, it, ev = C.c_double(0), C.c_int(0), C.c_int(0)
    r = lib().isdf_host_lbfgs_generic_ex(n, _p(x), C.byref(fx), C.cast(cfn, C.c_void_p), None, mem_size, past, delta, g_epsilon, max_iterations,
                                      *_ls_args(**{**LS_DEFAULTS, **ls}), C.byref(it), C.byref(ev))
    return dict(ret=r, x=x, f=fx.value, iterations=it.value, evaluations=ev.value, trace=trace)


EVAL_BATCH_T = C.CFUNCTYPE(None, C.c_void_p, C.c_int, C.POINTER(C.c_int), dp, dp, dp)   # lbfgs_eval_batch_t


def lbfgs_minimize_batch(fun, X0, mem_size=8, past=3, delta=1e-6, g_epsilon=1e-5, max_iterations=0, cancel_after=0, **ls):
    """fun(id, x) -> (f, grad) per instance; B instances advanced in lock step by the product's batched driver. ls: as lbfgs_minimize."""
    X = f(X0).copy()
    B, n = X.shape

    def cb(_inst, nb, ids, xp, fp, gp):
        xs = np.ctypeslib.as_array(xp, shape=(nb, n))
        fs = np.ctypeslib.as_array(fp, shape=(nb,))
        gs = np.ctypeslib.as_array(gp, shape=(nb, n))
        for q in range(nb):
            fv, gv = fun(ids[q], xs[q].copy())
            fs[q] = fv; gs[q] = gv
    cfn = EVAL_BATCH_T(cb)
    fx, ret, it, ev = np.zeros(B), np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32)
    ip = C.POINTER(C.c_int)
    Xf = X.reshape(-1)
    rounds = lib().isdf_host_lbfgs_batch_generic_ex(B, n, _p(Xf), _p(fx), ret.ctypes.data_as(ip), C.cast(cfn, C.c_void_p), None, mem_size, past,
                                                 delta, g_epsilon, max_iterations, *_ls_args(**{**LS_DEFAULTS, **ls}), int(cancel_after),
                                                 it.ctypes.data_as(ip), ev.ctypes.data_as(ip))
    X = Xf.reshape(B, n)
    return dict(rounds=rounds, ret=ret, x=X, f=fx, iterations=it, evaluations=ev)


def _p(a):
    return a.ctypes.data_as(dp)


def f(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def minco_forward(head, tail, inPs, T):
    T = f(T).reshape(-1)
    N = T.size
    h, t, ip = np.asfortranarray(f(head)), np.asfortranarray(f(tail)), np.asfortranarray(f(inPs).reshape(3, -1))
    co, gc, gt, e = np.zeros(18 * N), np.zeros(18 * N), np.zeros(N), C.c_double(0)
    lib().isdf_host_minco_forward(N, h.ctypes.data_as(dp), t.ctypes.data_as(dp), ip.ctypes.data_as(dp), _p(T), _p(co), C.byref(e), _p(gc), _p(gt))
    return co, e.value, gc, gt


def minco_backward(head, tail, inPs, T, gradC, gradT):
    T = f(T).reshape(-1)
    N = T.size
    h, t, ip = np.asfortranarray(f(head)), np.asfortranarray(f(tail)), np.asfortranarray(f(inPs).reshape(3, -1))
    gp, gt = np.zeros((3, N - 1), order="F"), np.zeros(N)
    lib().isdf_host_minco_backward(N, h.ctypes.data_as(dp), t.ctypes.data_as(dp), ip.ctypes.data_as(dp), _p(T), _p(f(gradC)), _p(f(gradT)),
                                   gp.ctypes.data_as(dp), _p(gt))
    return gp, gt


def tau_maps(tau):
    tau = f(tau)
    T, back = np.zeros_like(tau), np.zeros_like(tau)
    lib().isdf_host_tau_maps(_p(tau), tau.size, _p(T), _p(back))
    return T, back


def read_obj(path):
    """host/isdf_obj.hpp read_obj through its test hook -> (V [n,3] float64, F [m,3] int32)"""
    L = lib()
    nv, nf = C.c_int(0), C.c_int(0)
    if L.isdf_host_read_obj(path.encode(), None, 0, None, 0, C.byref(nv), C.byref(nf)) != 0:
        raise RuntimeError(f"read_obj failed for {path}")
    V, F = np.zeros((nv.value, 3)), np.zeros((nf.value, 3), dtype=np.int32)
    L.isdf_host_read_obj(path.encode(), V.ctypes.data_as(dp), nv.value, F.ctypes.data_as(C.POINTER(C.c_int32)), nf.value, C.byref(nv), C.byref(nf))
    return V, F
