"""CPU-side checks of the planning step's ABI: the ctypes mirrors of isdf_plan_params / isdf_plan_result / isdf_plan_info have the offsets
and sizes a g++-compiled probe of include/isdf.h reports, and the defaults need no device."""
import ctypes as C
import os
import subprocess
import tempfile
import isdf_b200 as I

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _fields(struct, prefix=""):
    """(dotted name, offset) of every field, nested structures flattened"""
    out = []
    for n, t in struct._fields_:
        off = getattr(struct, n).offset
        out.append((prefix + n, off))
        if isinstance(t, type) and issubclass(t, C.Structure):
            out += [(f, o + off) for f, o in _fields(t, prefix + n + ".")]
    return out


def _probe(structs):
    """{struct: (sizeof, {field: offsetof})} from a C++ program compiled against include/isdf.h"""
    lines = ['#include "isdf.h"', "#include <cstddef>", "#include <cstdio>", "int main() {"]
    for cname, py in structs:
        lines.append(f'  std::printf("{cname} sizeof %zu\\n", sizeof({cname}));')
        for f, _ in _fields(py):
            lines.append(f'  std::printf("{cname} {f} %zu\\n", offsetof({cname}, {f}));')
    lines.append("  return 0;\n}\n")
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "probe.cpp"), os.path.join(d, "probe")
        open(src, "w").write("\n".join(lines))
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([gxx, "-std=c++17", "-Wno-invalid-offsetof", "-I", os.path.join(ROOT, "include"), "-o", exe, src])
        out = subprocess.check_output([exe]).decode().split("\n")
    res = {}
    for l in out:
        if not l:
            continue
        cname, f, v = l.split()
        size, offs = res.setdefault(cname, [0, {}])
        if f == "sizeof":
            res[cname][0] = int(v)
        else:
            offs[f] = int(v)
    return res


def test_plan_struct_layouts_match_the_header():
    structs = [("isdf_plan_params", I.PlanParams), ("isdf_plan_result", I.PlanResult), ("isdf_plan_info", I.PlanInfo)]
    got = _probe(structs)
    for cname, py in structs:
        size, offs = got[cname]
        assert size == C.sizeof(py), cname
        assert offs == dict(_fields(py)), cname


def test_plan_default_params_without_a_context():
    lib = I.load_library()
    p = I.PlanParams()
    assert lib.isdf_plan_default_params(None, C.byref(p)) == 0
    cfg = I.default_config_values()
    assert p.parlength == 3.0 and p.rho == 20.0 and list(p.offset) == [0.0, 0.0, 0.0] and p.reserved_ == 0
    assert p.half_extent == cfg.kernel_size * cfg.occupancy_resolution / 3.0
    assert p.flags == I.PLAN_CERTIFY | I.PLAN_DYNAMICS
    assert p.backend.max_iterations == 10000 and p.midend.lbfgs.max_iterations == 100000 and p.midend.init_time == 2.5
    assert p.certify.clearance.pieces_per_traj == 0 and p.dynamics.pieces_per_traj == 0 and p.dynamics.vmax == cfg.vmax
    assert lib.isdf_plan_default_params(None, None) == -1


def test_plan_entry_points_refuse_a_null_context():
    lib = I.load_library()
    p = I.PlanParams()
    lib.isdf_plan_default_params(None, C.byref(p))
    res = (I.PlanResult * 2)()
    st, goals = (C.c_double * 3)(), (C.c_double * 6)()
    po = (C.c_int32 * 3)()
    assert lib.isdf_plan_batch(None, st, 2, goals, C.byref(p), 0, None, None, 0, po, None, None, res, None, None) == -1
    assert all(r.stage == I.PLAN_FAILED for r in res)
    assert lib.isdf_get_plan_info(None, None) == -1
    wo, pt = (C.c_int32 * 2)(), (C.c_int32 * 2)()
    assert lib.isdf_gather_obstacle_points_batch(None, 1, wo, None, 1.0, None, 0, None, pt, 0) == -1
