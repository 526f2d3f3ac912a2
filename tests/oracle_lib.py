"""ctypes binding of oracle/liboracle.so — TEST INFRASTRUCTURE (the CPU restatement of the reference hot path).
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs import this."""
import ctypes as C
import os
import subprocess
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
LIB = os.path.join(ORACLE_DIR, "liboracle.so")
REF_FWN = os.path.join(ORACLE_DIR, "_ref", "libref_fwn.so")
REF_FLAT = os.path.join(ORACLE_DIR, "_ref", "libref_flat.so")
REF_LBFGS = os.path.join(os.path.dirname(REF_FLAT), "libref_lbfgs.so")
REF_MINCO = os.path.join(os.path.dirname(REF_FLAT), "libref_minco.so")
REF_GRID = os.path.join(os.path.dirname(REF_FLAT), "libref_grid.so")

WN_EXACT, WN_BH, WN_RAW, WN_REF = 0, 1, 2, 3


def build(force=False):
    srcs = [os.path.join(ORACLE_DIR, f) for f in os.listdir(ORACLE_DIR) if f.endswith((".hpp", ".cpp"))]
    if force or not os.path.exists(LIB) or any(os.path.getmtime(s) > os.path.getmtime(LIB) for s in srcs):
        subprocess.check_call(["make", "-C", ORACLE_DIR, "liboracle.so"], stdout=subprocess.DEVNULL)
    if os.path.isdir("/root/reference/src/utils/include/igl") and not all(os.path.exists(p) for p in (REF_FWN, REF_FLAT, REF_LBFGS, REF_MINCO, REF_GRID)):
        subprocess.call(["make", "-C", ORACLE_DIR, "ref"], stdout=subprocess.DEVNULL)


class OrcConfig(C.Structure):
    _fields_ = [(n, C.c_double) for n in
                ["vehicle_mass", "grav_acc", "horiz_drag", "vert_drag", "paras_drag", "speed_eps", "vmax", "omgmax", "thetamax",
                 "weight_v", "weight_p", "weight_omg", "weight_theta", "smoothing_eps", "safety_hor", "occupancy_resolution"]] + \
               [(n, C.c_int32) for n in ["kernel_size", "integral_intervs", "threads_num", "flags"]]


_lib = None
dp = C.POINTER(C.c_double)


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB)
        L.orc_shape_create.restype = C.c_void_p
        L.orc_shape_create.argtypes = [C.c_int, dp, C.c_int, dp, dp]
        L.orc_shape_create_named.restype = C.c_void_p
        L.orc_shape_create_named.argtypes = [C.c_char_p, dp, dp]
        L.orc_shape_create_mesh.restype = C.c_void_p
        L.orc_shape_create_mesh.argtypes = [dp, C.c_int, C.POINTER(C.c_int32), C.c_int, dp, C.c_int]
        L.orc_shape_destroy.argtypes = [C.c_void_p]
        L.orc_shape_attach_ref_fwn.argtypes = [C.c_void_p, C.c_char_p]
        L.orc_shape_kind.argtypes = [C.c_void_p]
        L.orc_shape_params.argtypes = [C.c_void_p, dp]
        L.orc_shape_query.argtypes = [C.c_void_p, dp, C.c_int, dp, dp, C.c_int]
        L.orc_mesh_query.argtypes = [C.c_void_p, dp, C.c_int, dp, dp, dp, dp, dp]
        L.orc_flat_forward.argtypes = [C.POINTER(OrcConfig), dp, dp, dp, dp, dp]
        L.orc_flat_backward.argtypes = [C.POINTER(OrcConfig), dp, dp, dp, dp, dp, dp, dp, dp]
        L.orc_flat_forward_batch.argtypes = [C.POINTER(OrcConfig), C.c_int, dp, dp, dp, dp, dp]
        L.orc_flat_backward_batch.argtypes = [C.POINTER(OrcConfig), C.c_int, dp, dp, dp, dp, dp, dp, dp, dp]
        L.orc_eval_discrete.argtypes = [C.POINTER(OrcConfig), C.POINTER(C.c_uint8), C.c_int, C.c_int, C.c_int, dp, C.c_double,
                                        C.c_void_p, C.c_int, dp, dp, dp, dp, dp, C.POINTER(C.c_longlong), C.c_int, C.c_int, C.c_int]
        L.orc_eval_swept.argtypes = [C.POINTER(OrcConfig), C.c_void_p, C.c_int, dp, dp, C.c_int, dp, dp, dp, dp, dp, dp, dp,
                                     C.POINTER(C.c_longlong), C.c_int, dp, dp, dp]
        L.orc_eval_swept_ex.argtypes = L.orc_eval_swept.argtypes + [dp]
        L.orc_sv_coarse.argtypes = [C.POINTER(OrcConfig), C.c_void_p, C.c_int, dp, dp, C.c_int, dp, C.c_double, C.POINTER(C.c_uint32), C.c_int, dp,
                                    C.POINTER(C.c_int32)]
        L.orc_sdf_swept.restype = C.c_double
        L.orc_sdf_swept.argtypes = [C.POINTER(OrcConfig), C.c_void_p, C.c_int, dp, dp, dp, dp, dp]
        L.orc_points_in_aabb.argtypes = [C.POINTER(C.c_uint8), C.c_int, C.c_int, C.c_int, dp, C.c_double, dp, C.c_double, dp, C.c_int]
        L.orc_gather_obstacle_points.argtypes = [C.POINTER(C.c_uint8), C.c_int, C.c_int, C.c_int, dp, C.c_double, dp, C.c_int, C.c_double, dp, dp, C.c_int]
        L.orc_minco_forward.argtypes = [C.c_int, dp, dp, dp, dp, dp, dp, dp, dp]
        L.orc_minco_backward.argtypes = [C.c_int, dp, dp, dp, dp, dp, dp, dp, dp]
        u8p, ip, u32p = C.POINTER(C.c_uint8), C.POINTER(C.c_int32), C.POINTER(C.c_uint32)
        L.orc_frontend_create.restype = C.c_void_p
        L.orc_frontend_create.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int, u8p, C.c_int, C.c_int, C.c_int,
                                          C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.orc_frontend_destroy.argtypes = [C.c_void_p]
        L.orc_frontend_kernels.argtypes = [C.c_void_p, u8p]
        L.orc_frontend_feasibility.argtypes = [C.c_void_p, C.c_int, ip, u32p]
        L.orc_frontend_check.argtypes = [C.c_void_p, C.c_int, ip, dp, dp, u8p]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(dp) if a is not None else None


def f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def config_from(cfg):
    """copy any ctypes struct with the isdf_config layout (e.g. isdf_b200.Config) into an OrcConfig"""
    o = OrcConfig()
    assert C.sizeof(o) == C.sizeof(cfg)
    C.memmove(C.byref(o), C.byref(cfg), C.sizeof(o))
    return o


class Shape:
    def __init__(self, handle):
        assert handle, "oracle shape creation failed"
        self.h = C.c_void_p(handle)

    @staticmethod
    def named(name, rotate=None, trans=None):
        r = f64(rotate).reshape(9) if rotate is not None else None
        t = f64(trans).reshape(3) if trans is not None else None
        return Shape(lib().orc_shape_create_named(name.encode(), _p(r), _p(t)))

    @staticmethod
    def analytic(kind, params, rotate=None, trans=None):
        p = f64(params).reshape(-1)
        r = f64(rotate).reshape(9) if rotate is not None else None
        t = f64(trans).reshape(3) if trans is not None else None
        return Shape(lib().orc_shape_create(int(kind), _p(p) if p.size else None, p.size, _p(r), _p(t)))

    @staticmethod
    def mesh(V, F, poly_params=None, wn_mode=WN_EXACT):
        V = f64(V).reshape(-1, 3)
        F = np.ascontiguousarray(F, dtype=np.int32).reshape(-1, 3)
        pp = f64(poly_params).reshape(6) if poly_params is not None else None
        sh = Shape(lib().orc_shape_create_mesh(_p(V), V.shape[0], F.ctypes.data_as(C.POINTER(C.c_int32)), F.shape[0], _p(pp),
                                               WN_EXACT if wn_mode == WN_REF else wn_mode))
        if wn_mode == WN_REF:   # reference-faithful sign: s = 1 - 2 w with w from the reference-compiled FWN header (oracle/_ref)
            r = lib().orc_shape_attach_ref_fwn(sh.h, REF_FWN.encode())
            assert r == 0, f"cannot attach {REF_FWN} (rc {r}); build it with `make -C oracle ref` where /root/reference exists"
        return sh

    def kind(self):
        return lib().orc_shape_kind(self.h)

    def params(self):
        p = np.zeros(12)
        lib().orc_shape_params(self.h, _p(p))
        return p

    def query(self, p, what=2):
        p = f64(p).reshape(-1, 3)
        n = p.shape[0]
        sdf, grad = np.zeros(n), np.zeros((n, 3))
        lib().orc_shape_query(self.h, _p(p), n, _p(sdf), _p(grad), what)
        return sdf, grad

    def mesh_query(self, p, brute=True, winding=True):
        p = f64(p).reshape(-1, 3)
        n = p.shape[0]
        d2, d2b, c, we, wb = np.zeros(n), np.zeros(n), np.zeros((n, 3)), np.zeros(n), np.zeros(n)
        lib().orc_mesh_query(self.h, _p(p), n, _p(d2), _p(d2b) if brute else None, _p(c), _p(we) if winding else None, _p(wb) if winding else None)
        return dict(d2=d2, d2_brute=d2b, closest=c, w_exact=we, w_bh=wb)

    def __del__(self):
        try:
            lib().orc_shape_destroy(self.h)
        except Exception:
            pass


class FrontEnd:
    """oracle_frontend.hpp: the reference's attitude kernels, byte-packed map kernel, kernelConv<true>, BFS over attitudes."""

    def __init__(self, shape, occ, ks=13, res=1.0, max_roll=45.0, max_pitch=45.0, ang_res=9.0, front_end_safeh=0.0):
        occ = np.ascontiguousarray(occ, dtype=np.uint8)
        X, Y, Z = occ.shape
        xk, yk = C.c_int(0), C.c_int(0)
        self.shape = shape
        self.h = lib().orc_frontend_create(shape.h, max_roll, max_pitch, ang_res, front_end_safeh, res, ks, occ.ctypes.data_as(C.POINTER(C.c_uint8)), X, Y, Z,
                                           C.byref(xk), C.byref(yk))
        self.xk, self.yk, self.ks = xk.value, yk.value, ks

    def kernels(self):
        out = np.zeros(self.xk * self.yk * self.ks ** 3, dtype=np.uint8)
        lib().orc_frontend_kernels(self.h, out.ctypes.data_as(C.POINTER(C.c_uint8)))
        return out.reshape(self.xk * self.yk, self.ks, self.ks, self.ks)

    def feasibility(self, ind):
        ind = np.ascontiguousarray(ind, dtype=np.int32).reshape(-1, 3)
        out = np.zeros((ind.shape[0], 4), dtype=np.uint32)
        lib().orc_frontend_feasibility(self.h, ind.shape[0], ind.ctypes.data_as(C.POINTER(C.c_int32)), out.ctypes.data_as(C.POINTER(C.c_uint32)))
        return out

    def check(self, ind, father):
        ind = np.ascontiguousarray(ind, dtype=np.int32).reshape(-1, 3)
        father = f64(father).reshape(-1, 2)
        n = ind.shape[0]
        child, ok = np.zeros((n, 2)), np.zeros(n, dtype=np.uint8)
        lib().orc_frontend_check(self.h, n, ind.ctypes.data_as(C.POINTER(C.c_int32)), _p(father.reshape(-1)), _p(child.reshape(-1)),
                                 ok.ctypes.data_as(C.POINTER(C.c_uint8)))
        return child, ok.astype(bool)

    def __del__(self):
        try:
            lib().orc_frontend_destroy(self.h)
        except Exception:
            pass


def flat_forward(cfg, v, a, j):
    q, o = np.zeros(4), np.zeros(3)
    lib().orc_flat_forward(C.byref(cfg), _p(f64(v)), _p(f64(a)), _p(f64(j)), _p(q), _p(o))
    return q, o


def flat_backward(cfg, v, a, j, pos_grad, vel_grad, quat_grad, omg_grad):
    out = np.zeros(12)
    lib().orc_flat_backward(C.byref(cfg), _p(f64(v)), _p(f64(a)), _p(f64(j)), _p(f64(pos_grad)), _p(f64(vel_grad)), _p(f64(quat_grad)),
                            _p(f64(omg_grad)), _p(out))
    return out.reshape(4, 3)


def flat_forward_batch(cfg, v, a, j):
    v, a, j = f64(v).reshape(-1, 3), f64(a).reshape(-1, 3), f64(j).reshape(-1, 3)
    n = v.shape[0]
    q, o = np.zeros((n, 4)), np.zeros((n, 3))
    lib().orc_flat_forward_batch(C.byref(cfg), n, _p(v), _p(a), _p(j), _p(q), _p(o))
    return q, o


def flat_backward_batch(cfg, v, a, j, pos_grad, vel_grad, quat_grad, omg_grad):
    v, a, j = f64(v).reshape(-1, 3), f64(a).reshape(-1, 3), f64(j).reshape(-1, 3)
    n = v.shape[0]
    out = np.zeros((n, 12))
    lib().orc_flat_backward_batch(C.byref(cfg), n, _p(v), _p(a), _p(j), _p(f64(pos_grad).reshape(-1, 3)), _p(f64(vel_grad).reshape(-1, 3)),
                                  _p(f64(quat_grad).reshape(-1, 4)), _p(f64(omg_grad).reshape(-1, 3)), _p(out))
    return out


def grid_index(dims, bmin, res, pts, L=None, name="orc_grid_index"):
    """getGridIndex / getGridCubeCenter / isInMap for n points: the oracle's (default) or, with L = RefGrid().L, the reference-compiled grid's"""
    L = L or lib()
    pts = f64(pts).reshape(-1, 3)
    n = pts.shape[0]
    idx, ctr, inm = np.zeros((n, 3), dtype=np.int32), np.zeros((n, 3)), np.zeros(n, dtype=np.int32)
    fn = getattr(L, name)
    fn.argtypes = [C.c_int, C.c_int, C.c_int, dp, C.c_double, C.c_int, dp, C.POINTER(C.c_int), dp, C.POINTER(C.c_int)]
    r = fn(int(dims[0]), int(dims[1]), int(dims[2]), _p(f64(bmin)), float(res), n, _p(pts), idx.ctypes.data_as(C.POINTER(C.c_int)), _p(ctr),
           inm.ctypes.data_as(C.POINTER(C.c_int)))
    assert r == 0, "grid dimensions do not survive createGridMap's ceil((max - min) / res)"
    return idx, ctr, inm


class RefGrid:
    """oracle/_ref/libref_grid.so: the reference's own map_manager/src/Gridmap3D.cpp compiled unmodified (eager Eigen stand-in, ROS stand-ins) —
    kind "reference"."""

    def __init__(self):
        self.L = C.CDLL(REF_GRID)
        self.L.ref_points_in_aabb.argtypes = [C.POINTER(C.c_uint8), C.c_int, C.c_int, C.c_int, dp, C.c_double, dp, C.c_double, dp, C.c_int]

    def index(self, dims, bmin, res, pts):
        return grid_index(dims, bmin, res, pts, L=self.L, name="ref_grid_index")

    def points_in_aabb(self, occ, bmin, res, centre, half, cap=100000):
        occ = np.ascontiguousarray(occ, dtype=np.uint8)
        X, Y, Z = occ.shape
        out = np.zeros((cap, 3))
        n = self.L.ref_points_in_aabb(occ.ctypes.data_as(C.POINTER(C.c_uint8)), X, Y, Z, _p(f64(bmin)), float(res), _p(f64(centre)), float(half), _p(out), cap)
        return out[:max(0, min(n, cap))].copy(), n


class RefMinco:
    """oracle/_ref/libref_minco.so: the reference's own utils/minco.hpp (BandedSystem, MINCO_S3NU) compiled unmodified against the eager
    Eigen stand-in — kind "reference". Same calling convention as minco_forward / minco_backward below."""

    def __init__(self):
        self.L = C.CDLL(REF_MINCO)
        self.L.ref_minco_forward.argtypes = [C.c_int, dp, dp, dp, dp, dp, dp, dp, dp]
        self.L.ref_minco_backward.argtypes = [C.c_int, dp, dp, dp, dp, dp, dp, dp, dp]
        self.L.ref_minco_trajectory.argtypes = [C.c_int, dp, dp, dp, dp, dp, dp]
        self.L.ref_traj_eval.argtypes = [C.c_int, dp, dp, dp, dp, C.c_int, dp, dp, C.POINTER(C.c_int), dp, dp]

    @staticmethod
    def _in(head, tail, inPs, T):
        T = f64(T).reshape(-1)
        return T.size, np.asfortranarray(f64(head)), np.asfortranarray(f64(tail)), np.asfortranarray(f64(inPs).reshape(3, -1)), T

    def forward(self, head, tail, inPs, T):
        N, h, t, ip, T = self._in(head, tail, inPs, T)
        co, gc, gt, e = np.zeros(18 * N), np.zeros(18 * N), np.zeros(N), C.c_double(0)
        self.L.ref_minco_forward(N, h.ctypes.data_as(dp), t.ctypes.data_as(dp), ip.ctypes.data_as(dp), _p(T), _p(co), C.byref(e), _p(gc), _p(gt))
        return co, e.value, gc, gt

    def backward(self, head, tail, inPs, T, gradC, gradT):
        N, h, t, ip, T = self._in(head, tail, inPs, T)
        gp, gt = np.zeros((3, N - 1), order="F"), np.zeros(N)
        self.L.ref_minco_backward(N, h.ctypes.data_as(dp), t.ctypes.data_as(dp), ip.ctypes.data_as(dp), _p(T), _p(f64(gradC)), _p(f64(gradT)),
                                  gp.ctypes.data_as(dp), _p(gt))
        return gp, gt

    def traj_eval(self, head, tail, inPs, T, times):
        """MINCO -> the reference's Trajectory<5> -> getPos_Vel_Acc_Jerk / locatePieceIdx at absolute times"""
        N, h, t, ip, T = self._in(head, tail, inPs, T)
        times = f64(times).reshape(-1)
        out, piece, tloc, total = np.zeros((times.size, 12)), np.zeros(times.size, dtype=np.int32), np.zeros(times.size), C.c_double(0)
        self.L.ref_traj_eval(N, h.ctypes.data_as(dp), t.ctypes.data_as(dp), ip.ctypes.data_as(dp), _p(T), times.size, _p(times), _p(out),
                             piece.ctypes.data_as(C.POINTER(C.c_int)), _p(tloc), C.byref(total))
        return out, piece, tloc, total.value

    def trajectory(self, head, tail, inPs, T):
        N, h, t, ip, T = self._in(head, tail, inPs, T)
        dur, cm = np.zeros(N), np.zeros(18 * N)
        self.L.ref_minco_trajectory(N, h.ctypes.data_as(dp), t.ctypes.data_as(dp), ip.ctypes.data_as(dp), _p(T), _p(dur), _p(cm))
        return dur, cm.reshape(N, 6, 3).transpose(0, 2, 1)          # per piece 3 x 6, highest power first


class RefLbfgs:
    """oracle/_ref/libref_lbfgs.so: the reference's own utils/lbfgs.hpp (lbfgs_optimize, line_search_lewisoverton) compiled unmodified
    against the eager dynamic-vector Eigen stand-in (left-to-right reductions) — kind "reference"."""
    EVAL_T = C.CFUNCTYPE(C.c_double, C.c_void_p, C.c_int, dp, dp)

    def __init__(self):
        self.L = C.CDLL(REF_LBFGS)
        self.L.ref_lbfgs_optimize.argtypes = [C.c_int, dp, dp, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int, C.c_double,
                                              C.POINTER(C.c_long)]
        self.L.ref_lbfgs_optimize.restype = C.c_int
        # the full parameter set; a library built from an older wrapper has only ref_lbfgs_optimize
        self.full = hasattr(self.L, "ref_lbfgs_optimize_ex")
        if self.full:
            self.L.ref_lbfgs_optimize_ex.argtypes = self.L.ref_lbfgs_optimize.argtypes[:-1] + [C.c_int, C.c_double, C.c_double, C.c_double, C.c_double,
                                                                                               C.POINTER(C.c_long)]
            self.L.ref_lbfgs_optimize_ex.restype = C.c_int

    def minimize(self, fun, x0, mem_size=8, past=3, delta=1e-6, g_epsilon=1e-5, max_iterations=0, min_step=1e-32, max_linesearch=64, max_step=1e20,
                 f_dec_coeff=1e-4, cautious_factor=1e-6, machine_prec=1e-16):
        """fun(x) -> (f, grad); returns ret, x, f, evaluations and the list of every point the optimiser evaluated"""
        x = f64(x0).copy()
        n = x.size
        trace = []

        def cb(_u, nn, xp, gp):
            xv = np.ctypeslib.as_array(xp, shape=(nn,)).copy()
            trace.append(xv)
            fv, gv = fun(xv.copy())
            np.ctypeslib.as_array(gp, shape=(nn,))[:] = gv
            return float(fv)
        cfn = self.EVAL_T(cb)
        fx, ev = C.c_double(0), C.c_long(0)
        ls = (max_linesearch, max_step, f_dec_coeff, cautious_factor, machine_prec)
        args = (n, _p(x), C.byref(fx), C.cast(cfn, C.c_void_p), None, mem_size, past, delta, g_epsilon, max_iterations, min_step)
        if self.full:
            r = self.L.ref_lbfgs_optimize_ex(*args, *ls, C.byref(ev))
        elif ls == (64, 1e20, 1e-4, 1e-6, 1e-16):    # lbfgs_parameter_t's defaults, what ref_lbfgs_optimize sets
            r = self.L.ref_lbfgs_optimize(*args, C.byref(ev))
        else:
            raise RuntimeError(f"{REF_LBFGS} predates ref_lbfgs_optimize_ex: rebuild it (make -C oracle ref) to set the line-search parameters")
        return dict(ret=r, x=x, f=fx.value, evaluations=ev.value, trace=trace)


class RefFlat:
    """oracle/_ref/libref_flat.so: the reference's own utils/flatness.hpp (optimizated_forward x2, backwardthreadsafe) compiled
    unmodified against the element-access-only Eigen stand-in — kind "reference"."""

    def __init__(self, cfg):
        self.L = C.CDLL(REF_FLAT)
        self.L.ref_flat_forward_quat.argtypes = [dp, C.c_int, dp, dp, dp, dp]
        self.L.ref_flat_forward_quat_omg.argtypes = [dp, C.c_int, dp, dp, dp, dp, dp]
        self.L.ref_flat_backward.argtypes = [dp, C.c_int, dp, dp, dp, dp, dp, dp, dp, dp]
        self.par = np.array([cfg.vehicle_mass, cfg.grav_acc, cfg.horiz_drag, cfg.vert_drag, cfg.paras_drag, cfg.speed_eps], dtype=np.float64)

    def forward_quat(self, v, a, j):
        v, a, j = f64(v).reshape(-1, 3), f64(a).reshape(-1, 3), f64(j).reshape(-1, 3)
        q = np.zeros((v.shape[0], 4))
        self.L.ref_flat_forward_quat(_p(self.par), v.shape[0], _p(v), _p(a), _p(j), _p(q))
        return q

    def forward(self, v, a, j):
        v, a, j = f64(v).reshape(-1, 3), f64(a).reshape(-1, 3), f64(j).reshape(-1, 3)
        q, o = np.zeros((v.shape[0], 4)), np.zeros((v.shape[0], 3))
        self.L.ref_flat_forward_quat_omg(_p(self.par), v.shape[0], _p(v), _p(a), _p(j), _p(q), _p(o))
        return q, o

    def backward(self, v, a, j, pos_grad, vel_grad, quat_grad, omg_grad):
        v, a, j = f64(v).reshape(-1, 3), f64(a).reshape(-1, 3), f64(j).reshape(-1, 3)
        out = np.zeros((v.shape[0], 12))
        self.L.ref_flat_backward(_p(self.par), v.shape[0], _p(v), _p(a), _p(j), _p(f64(pos_grad).reshape(-1, 3)), _p(f64(vel_grad).reshape(-1, 3)),
                                 _p(f64(quat_grad).reshape(-1, 4)), _p(f64(omg_grad).reshape(-1, 3)), _p(out))
        return out


def ref_flat_available():
    return os.path.exists(REF_FLAT)


def eval_discrete(cfg, occ, bmin, res, shape, T, coeffs, use_omp=False, rank=0, world=1):
    T = f64(T).reshape(-1)
    N = T.size
    Cc = f64(coeffs).reshape(-1)
    gC, gT, cost, npairs = np.zeros(18 * N), np.zeros(N), C.c_double(0), C.c_longlong(0)
    if occ is not None:
        occ = np.ascontiguousarray(occ, dtype=np.uint8)
        X, Y, Z = occ.shape
        op = occ.ctypes.data_as(C.POINTER(C.c_uint8))
    else:
        X = Y = Z = 0
        op = None
    b = f64(bmin).reshape(3)
    lib().orc_eval_discrete(C.byref(cfg), op, X, Y, Z, _p(b), float(res), shape.h if shape is not None else None, N, _p(T), _p(Cc),
                            C.byref(cost), _p(gC), _p(gT), C.byref(npairs), int(use_omp), rank, world)
    return cost.value, gC, gT, npairs.value


def eval_swept(cfg, shape, T, coeffs, pts, tstar=None, use_omp=False, given=None, prev_duration=0.0):
    """prev_duration: the persisted trajectory duration before this evaluation (a fresh SweptVolumeManager has 0); the result's
    "duration" is the one after it (quirk Q14: a trajectory of 300 s or longer keeps the previous one)"""
    T = f64(T).reshape(-1)
    N = T.size
    Cc = f64(coeffs).reshape(-1)
    pts = f64(pts).reshape(-1, 3)
    P = pts.shape[0]
    ts = np.zeros(P) if tstar is None else f64(tstar).copy()
    gC, gT, cost, nsdf = np.zeros(18 * N), np.zeros(N), C.c_double(0), C.c_longlong(0)
    sdf, grel = np.zeros(P), np.zeros((P, 3))
    g_t = g_s = g_g = None
    if given is not None:
        g_t, g_s, g_g = f64(given[0]), f64(given[1]), f64(given[2]).reshape(-1)
    dur = C.c_double(prev_duration)
    lib().orc_eval_swept_ex(C.byref(cfg), shape.h, N, _p(T), _p(Cc), P, _p(pts), _p(ts), C.byref(cost), _p(gC), _p(gT), _p(sdf), _p(grel),
                            C.byref(nsdf), int(use_omp), _p(g_t), _p(g_s), _p(g_g), C.byref(dur))
    return dict(cost=cost.value, gradC=gC, gradT=gT, tstar=ts, sdf=sdf, grel=grel, nsdf=nsdf.value, duration=dur.value)


def sv_coarse(cfg, shape, T, coeffs, pts, prev_duration=0.0, words=48):
    """the swept-volume search's coarse decisions per point: (nc, bits (P, words) uint32, margin (P,), carried (P,)) — see orc_sv_coarse"""
    T = f64(T).reshape(-1)
    Cc = f64(coeffs).reshape(-1)
    pts = f64(pts).reshape(-1, 3)
    P = pts.shape[0]
    bits, margin, carried = np.zeros((P, words), dtype=np.uint32), np.zeros(P), np.zeros(P, dtype=np.int32)
    nc = lib().orc_sv_coarse(C.byref(cfg), shape.h, T.size, _p(T), _p(Cc), P, _p(pts), float(prev_duration),
                             bits.ctypes.data_as(C.POINTER(C.c_uint32)), words, _p(margin), carried.ctypes.data_as(C.POINTER(C.c_int32)))
    return nc, bits, margin, carried


def points_in_aabb(occ, bmin, res, centre, half, cap=100000):
    occ = np.ascontiguousarray(occ, dtype=np.uint8)
    X, Y, Z = occ.shape
    out = np.zeros((cap, 3))
    n = lib().orc_points_in_aabb(occ.ctypes.data_as(C.POINTER(C.c_uint8)), X, Y, Z, _p(f64(bmin)), float(res), _p(f64(centre)), float(half), _p(out), cap)
    return out[:min(n, cap)].copy(), n


def gather_obstacle_points(occ, bmin, res, wps, half, offset=(0, 0, 0), cap=2000000):
    occ = np.ascontiguousarray(occ, dtype=np.uint8)
    X, Y, Z = occ.shape
    wps = f64(wps).reshape(-1, 3)
    out = np.zeros((cap, 3))
    n = lib().orc_gather_obstacle_points(occ.ctypes.data_as(C.POINTER(C.c_uint8)), X, Y, Z, _p(f64(bmin)), float(res), _p(wps), wps.shape[0],
                                         float(half), _p(f64(offset)), _p(out), cap)
    return out[:min(n, cap)].copy(), n


def minco_forward(head, tail, inPs, T):
    """head/tail: 3x3 with columns pos, vel, acc; inPs 3 x (N-1). Returns coeffs (flat col-major), energy, dE/dC, dE/dT."""
    T = f64(T).reshape(-1)
    N = T.size
    h, t = np.asfortranarray(f64(head)), np.asfortranarray(f64(tail))
    ip = np.asfortranarray(f64(inPs).reshape(3, -1))
    co, gc, gt, e = np.zeros(18 * N), np.zeros(18 * N), np.zeros(N), C.c_double(0)
    lib().orc_minco_forward(N, h.ctypes.data_as(dp), t.ctypes.data_as(dp), ip.ctypes.data_as(dp), _p(T), _p(co), C.byref(e), _p(gc), _p(gt))
    return co, e.value, gc, gt


def traj_eval(T, coeffs, times):
    """the oracle's Trajectory evaluation on a 6N x 3 column-major coefficient block"""
    T, coeffs, times = f64(T).reshape(-1), f64(coeffs).reshape(-1), f64(times).reshape(-1)
    L = lib()
    L.orc_traj_eval.argtypes = [C.c_int, dp, dp, C.c_int, dp, dp, C.POINTER(C.c_int), dp, dp]
    out, piece, tloc, total = np.zeros((times.size, 12)), np.zeros(times.size, dtype=np.int32), np.zeros(times.size), C.c_double(0)
    L.orc_traj_eval(T.size, _p(T), _p(coeffs), times.size, _p(times), _p(out), piece.ctypes.data_as(C.POINTER(C.c_int)), _p(tloc), C.byref(total))
    return out, piece, tloc, total.value


def minco_backward(head, tail, inPs, T, gradC, gradT):
    T = f64(T).reshape(-1)
    N = T.size
    h, t = np.asfortranarray(f64(head)), np.asfortranarray(f64(tail))
    ip = np.asfortranarray(f64(inPs).reshape(3, -1))
    gp, gt = np.zeros((3, N - 1), order="F"), np.zeros(N)
    lib().orc_minco_backward(N, h.ctypes.data_as(dp), t.ctypes.data_as(dp), ip.ctypes.data_as(dp), _p(T), _p(f64(gradC)), _p(f64(gradT)),
                             gp.ctypes.data_as(dp), _p(gt))
    return gp, gt


class RefFwn:
    """oracle/_ref/libref_fwn.so: the reference's own FastWindingNumberForSoups.h compiled as a known-answer source."""

    def __init__(self, V, F, order=2):
        self.L = C.CDLL(REF_FWN)
        self.L.ref_fwn_create.restype = C.c_void_p
        self.L.ref_fwn_create.argtypes = [dp, C.c_int, C.POINTER(C.c_int32), C.c_int, C.c_int]
        self.L.ref_fwn_query.argtypes = [C.c_void_p, dp, C.c_int, C.c_double, dp]
        self.L.ref_fwn_destroy.argtypes = [C.c_void_p]
        self.V = f64(V).reshape(-1, 3)
        self.F = np.ascontiguousarray(F, dtype=np.int32).reshape(-1, 3)
        self.h = C.c_void_p(self.L.ref_fwn_create(_p(self.V), self.V.shape[0], self.F.ctypes.data_as(C.POINTER(C.c_int32)), self.F.shape[0], order))

    def query(self, q, accuracy_scale=2.0):
        q = f64(q).reshape(-1, 3)
        w = np.zeros(q.shape[0])
        self.L.ref_fwn_query(self.h, _p(q), q.shape[0], accuracy_scale, _p(w))
        return w

    def __del__(self):
        try:
            self.L.ref_fwn_destroy(self.h)
        except Exception:
            pass


def ref_fwn_available():
    return os.path.exists(REF_FWN)
