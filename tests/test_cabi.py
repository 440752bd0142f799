"""The C-ABI shared libraries load on a CPU-only box, type every function their headers declare exactly as declared, take every
wrapper's arguments against those types, and refuse to compute without a CUDA device (no CPU fallback)."""
import ctypes as C
import os
import re
from types import SimpleNamespace

import numpy as np
import pytest

from obca_b200 import _lib, parking as pk, quadcopter as qc, scenarios
from obca_b200.planner import a_star_3d, device, native

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADERS = ("obca.h", "obca_planner.h")


def _source(header):
    return re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", header)).read(), flags=re.S)


def _declared(header):
    return sorted(set(re.findall(r"\b(obca_[a-z_0-9]+)\s*\(", _source(header))))


def _prototype(header, name):
    """(restype, argtypes) of the function `name` as its declaration in the header reads."""
    m = re.search(r"(int|double|void|const char\*) " + name + r"\(([^;]*)\);", _source(header))
    assert m, f"declaration of {name} missing from include/{header}"
    ty = []
    for a in m.group(2).split(","):
        a = " ".join(a.split())
        if a != "void":
            ty.append(C.c_void_p if "*" in a else C.c_double if a.startswith("double ") else C.c_longlong if a.startswith("long long ")
                      else C.c_int if a.startswith("int ") else a)
    return {"int": C.c_int, "double": C.c_double, "void": None, "const char*": C.c_char_p}[m.group(1)], ty


def test_header_symbols_exported():
    import obca_b200
    lib = obca_b200.lib()
    names = _declared("obca.h")
    assert "obca_parking_solve_batch" in names and "obca_dualmultws_batch" in names and len(names) >= 8
    assert sorted(obca_b200._lib.SYMBOLS) == names      # each of them typed by test_binding_types_match_the_header
    assert lib.obca_version() == 200


@pytest.mark.parametrize("header,name", [pytest.param(h, n, id=n) for h in HEADERS for n in _declared(h)])
def test_binding_types_match_the_header(header, name):
    """The loaded library types every function its header declares, exactly as the declaration reads."""
    restype, argtypes = _prototype(header, name)
    f = getattr(_lib.lib() if header == "obca.h" else native.lib(), name)
    assert f.restype is restype and list(f.argtypes) == argtypes, (f.restype, f.argtypes)


def test_header_reader_refuses_what_it_cannot_type(tmp_path):
    h = tmp_path / "api.h"
    ok = "/* f(float) */\n#define K(x) (x)\nint ok(const float* a, long long n);\nvoid none(void);\n"
    h.write_text(ok)
    assert _lib.prototypes(str(h), _lib.ObcaError) == {"ok": (C.c_int, [C.c_void_p, C.c_longlong]), "none": (None, [])}
    for bad, what in (("int bad(int n, float x);", "'float x'"), ("float* bad(void);", "'float \\*'")):
        h.write_text(ok + bad)
        with pytest.raises(_lib.ObcaError, match="bad: .*" + what):
            _lib.prototypes(str(h), _lib.ObcaError)
    with pytest.raises(_lib.ObcaError, match="missing.h"):
        _lib.prototypes(str(tmp_path / "missing.h"), _lib.ObcaError)


def test_default_opts_match_reference_call_site():
    """ParkingSignedDist.jl:41-43: tol=1e-5, max_iter=200, min_hessian_perturbation=1e-12."""
    import obca_b200
    o = obca_b200.default_opts()
    assert o.tol == 1e-5 and o.max_iter == 200 and o.dw_min == 1e-12 and o.mu_init == 0.1 and o.retry == 1
    assert o.kappa_eps == 10.0 and o.tau_min == 0.99 and o.gamma_theta == 1e-5


def test_no_cpu_fallback():
    import obca_b200
    from obca_b200 import parking, scenarios
    if obca_b200.lib().obca_device_count() > 0:
        pytest.skip("CUDA device present")
    sc = scenarios.reverse_parking_batch(1, 20, 0)
    with pytest.raises(obca_b200.ObcaError, match="no CUDA device"):
        parking.parking_solve_batch(sc["x0"], sc["xF"], 20, sc["Ts"], sc["L"], sc["ego"], sc["XYbounds"], 3, sc["vOb"],
                                    sc["A"], sc["b"], sc["rx"], sc["ry"], sc["ryaw"], 0, sc["xWS"], sc["uWS"])
    with pytest.raises(obca_b200.ObcaError):
        parking.dualmultws_batch(20, 3, sc["vOb"], sc["A"], sc["b"], sc["rx"], sc["ry"], sc["ryaw"], sc["ego"])


@pytest.fixture(scope="module")
def tiny():
    """Tiny valid arguments for the wrappers: one parking and one quadcopter problem at N = 20, and two of each at N = 20 and 24."""
    N, Ns = 20, [20, 24]
    s, m = scenarios.reverse_parking_batch(1, N), scenarios.reverse_parking_mixed_batch(2, Ns=Ns)
    q, qm = scenarios.quadcopter_batch(1, N), scenarios.quadcopter_mixed_batch(2, Ns=Ns)
    V, nOb = int(s["vOb"].sum()), s["nOb"]
    shape = (s["Ts"], s["L"], s["ego"], s["XYbounds"], nOb, s["vOb"], s["A"], s["b"])
    pt = lambda n: (np.zeros((4, n + 1)), np.zeros((2, n)), np.zeros((V, n + 1)), np.zeros((4 * nOb, n + 1)), np.ones(n + 1))
    qt = lambda n: (np.zeros((12, n + 1)), np.zeros((4, n)), np.ones(n + 1), np.zeros((30, n + 1)))
    lists = lambda f: [list(a) for a in zip(*map(f, Ns))]
    obst = shape[4:] + shape[2:4]
    plan = (s["x0"], s["xF"], *native.obstacle_points("backwards"), 0.6)
    return SimpleNamespace(
        ego=s["ego"],
        one=(s["x0"][0], s["xF"], N, *shape, s["rx"][0], s["ry"][0], s["ryaw"][0], 0, s["xWS"][0], s["uWS"][0]),
        planned=(s["x0"], s["xF"], [{k: s[k][0] for k in ("rx", "ry", "ryaw", "xWS", "uWS")} | dict(N=N)], *shape),
        dualws=(N, nOb, s["vOb"], s["A"], s["b"], s["rx"][0], s["ry"][0], s["ryaw"][0]),
        check=(s["x0"], s["xF"], N, *shape, *[a[None] for a in pt(N)], 0, 1),
        check_mixed=(m["x0"], m["xF"], m["Ns"], *shape, *lists(pt), 0, 1),
        constraints=(s["x0"][0], s["xF"], N, *shape, *pt(N), 0, 1),
        qsolve=(q["x0"], q["xF"], N, q["Ts"], q["R"], q["obs"], q["xWS"]),
        qmixed=(qm["x0"], qm["xF"], qm["Ns"], qm["Ts"], qm["R"], qm["obs"], qm["xWS"]),
        qone=(q["x0"][0], q["xF"][0], N, q["Ts"], q["R"], *q["obs"], q["xWS"][0], np.zeros((4, N)), 1.0),
        qcheck=(*[a[None] for a in qt(N)[:3]], q["x0"], q["xF"], q["Ts"], qt(N)[3][None], q["obs"], q["R"]),
        qcheck_mixed=(*lists(qt)[:3], qm["x0"], qm["xF"], qm["Ns"], qm["Ts"], lists(qt)[3], qm["obs"], qm["R"]),
        qconstr=(*qt(N)[:3], q["x0"][0], q["xF"][0], q["Ts"], qt(N)[3], *q["obs"], q["R"]),
        plan=plan, qplan=native.quadcopter_problem(q["x0"], q["xF"]), flow=plan + obst, batch=(s["x0"], s["xF"], *obst),
        qflow_raw=(q["x0"], q["xF"], *a_star_3d.quadcopter_environment(), 1.0, q["Ts80"], q["R"], q["obs"]))


# the public wrappers of parking, quadcopter and planner.device that no other test calls through the library, and the arguments of
# `tiny` they get (parking.eval_batch stages its inputs with torch's CUDA before it reaches the library)
MODULES = {"parking": pk, "quadcopter": qc, "device": device}
CALLS = {"parking.ParkingSignedDist": "one", "parking.ParkingDist": "one", "parking.parking_solve_planned": "planned",
         "parking.DualMultWS": "dualws", "parking.check_parking_batch": "check", "parking.check_parking_mixed": "check_mixed",
         "parking.ParkingConstraints": "constraints", "quadcopter.quadcopter_solve_batch": "qsolve",
         "quadcopter.quadcopter_solve_mixed": "qmixed", "quadcopter.QuadcopterSignedDist": "qone", "quadcopter.QuadcopterDist": "qone",
         "quadcopter.check_quadcopter_batch": "qcheck", "quadcopter.check_quadcopter_mixed": "qcheck_mixed",
         "quadcopter.constrSatisfaction": "qconstr", "device.plan_raw": "plan", "device.plan_goals_raw": "plan",
         "device.plan_quadcopter_raw": "qplan", "device.plan_solve_goals": "flow", "device.plan_solve_goals_both": "flow",
         "device.plan_solve_batch": "batch", "device.plan_solve_quadcopter_raw": "qflow_raw",
         "device.plan_solve_quadcopter_both_raw": "qflow_raw"}


@pytest.mark.parametrize("wrapper", CALLS)
def test_wrapper_arguments_pass_the_binding_types(wrapper, tiny, monkeypatch):
    """ctypes accepts every argument the wrapper passes against the types read from the header, and the library then stops at the
    missing device."""
    import obca_b200
    if obca_b200.lib().obca_device_count() > 0:
        pytest.skip("CUDA device present")
    monkeypatch.setattr(pk, "ego", tiny.ego)      # DualMultWS reads the module's global, as the reference does
    module, name = wrapper.split(".")
    with pytest.raises(obca_b200.ObcaError, match="no CUDA device"):
        getattr(MODULES[module], name)(*getattr(tiny, CALLS[wrapper]))


def test_argument_errors():
    import obca_b200
    lib = obca_b200.lib()
    rc = lib.obca_parking_solve_batch(C.c_int(0), C.c_int(80), C.c_int(3), *([None] * 5), C.c_double(0.6), C.c_double(2.7),
                                      *([None] * 9), C.c_int(0), C.c_int(1), None, *([None] * 10))
    assert rc == -1
    assert b"null" in lib.obca_last_error()


def test_product_does_not_import_oracle():
    """Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline may touch oracle/."""
    for dp, _, files in os.walk(os.path.join(ROOT, "obca_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dp, f)).read()
                assert "import oracle" not in txt and "from oracle" not in txt and "oracle/" not in txt.replace(
                    "oracle/ipm_ref.py is the independent restatement", ""), f
