"""CPU-side checks of the drop-in boundary: the C-ABI library loads and exports every symbol include/ovp.h declares, and it
refuses to run without a CUDA device (no CPU fallback).  No compute call is made here."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    txt = open(os.path.join(ROOT, "include", "ovp.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(ovp_[a-z0-9_]+)\s*\(", txt)))


def test_library_exports_every_declared_symbol():
    from ov_plane_b200 import api
    if not os.path.exists(api.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    lib = ctypes.CDLL(api.LIB_PATH)
    syms = declared_symbols()
    assert len(syms) >= 60
    missing = [s for s in syms if not hasattr(lib, s)]
    assert not missing, missing


def _exported(path, prefix):
    import subprocess
    out = subprocess.check_output(["nm", "-D", "--defined-only", path]).decode()
    return sorted(set(re.findall(r"\b T (%s[a-z0-9_]+)$" % prefix, out, flags=re.M)))


def test_libraries_export_exactly_the_declared_symbols():
    """libovp.so exports exactly the symbols of include/ovp.h: no test / tuning hooks (those live in libovp_debug.so and are
    declared in include/ovp_debug.h); libovp_debug.so exports exactly the hooks include/ovp_debug.h declares, and the whole ABI."""
    from ov_plane_b200 import api
    exported = _exported(api.LIB_PATH, "ovp_")
    assert exported == declared_symbols(), sorted(set(exported) ^ set(declared_symbols()))
    txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "ovp_debug.h")).read(), flags=re.S)
    hooks = sorted(set(re.findall(r"\b(ovp_debug_[a-z0-9_]+)\s*\(", txt)))
    assert hooks
    dbg_hooks = _exported(api.DEBUG_LIB_PATH, "ovp_debug_")
    assert dbg_hooks == hooks, sorted(set(dbg_hooks) ^ set(hooks))
    dbg = ctypes.CDLL(api.DEBUG_LIB_PATH)
    assert not [s for s in declared_symbols() if not hasattr(dbg, s)]


def test_no_cpu_fallback():
    """Without a CUDA device the product path must fail loudly, not fall back."""
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("a GPU is present")
    except ImportError:
        pass
    from ov_plane_b200 import api, synth
    S = synth.make_scenario("tiny_points")
    with pytest.raises(api.OvpError):
        api.Context(S.options, device=0, max_state=128, max_meas_rows=1024)


def test_product_does_not_reference_oracle():
    """The oracle is test infrastructure: nothing under ov_plane_b200/ or include/ may mention it."""
    bad = []
    for base in ("ov_plane_b200", "include"):
        for dp, _, fs in os.walk(os.path.join(ROOT, base)):
            for f in fs:
                if f.endswith((".py", ".cu", ".cuh", ".h", ".inc", ".hpp", ".cpp")):
                    t = open(os.path.join(dp, f), errors="ignore").read()
                    if re.search(r"liboracle|oracle_backend|oracle/|import oracle|orc_", t):
                        bad.append(os.path.join(dp, f))
    assert not bad, bad


# ---- UpdaterHelper::get_feature_jacobian_representation: context-free host helper, testable without a GPU -------------------------
def _rep_call(lib, fn, rep, do_fej, pG, pGf, pA, anc, ancf, cal):
    import ctypes as C
    Hf, Ha, Hc = np.zeros(9), np.zeros(18), np.zeros(18)
    hfc, has = C.c_int(0), C.c_int(0)
    p = lambda a: np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(C.c_void_p)
    keep = [np.ascontiguousarray(a, dtype=np.float64) for a in (pG, pGf, pA, anc, ancf, cal)]
    st = getattr(lib, fn)(rep, do_fej, *[k.ctypes.data_as(C.c_void_p) for k in keep], Hf.ctypes.data_as(C.c_void_p), C.byref(hfc),
                          Ha.ctypes.data_as(C.c_void_p), Hc.ctypes.data_as(C.c_void_p), C.byref(has))
    assert st == 0
    return Hf[:3 * hfc.value].reshape((3, hfc.value), order="F"), Ha.reshape((3, 6), order="F"), Hc.reshape((3, 6), order="F"), has.value


def test_feature_jacobian_representation_vs_oracle_and_numerical_derivative():
    import ctypes as C
    import oracle_backend as ob
    from ov_plane_b200 import api, jpl
    lib = C.CDLL(api.LIB_PATH)        # no context: the helper is pure host algebra
    orc = C.CDLL(ob._LIB)
    rng = np.random.default_rng(11)

    def rand_pose():
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        if q[3] < 0:
            q = -q
        return np.concatenate([q, rng.normal(size=3)])

    def to_lambda(rep, pG, pA):
        if rep == 0:
            return pG.copy()
        p = pG if rep == 1 else pA
        if rep in (1, 3):
            rho = 1 / np.linalg.norm(p)
            return np.array([np.arctan2(p[1], p[0]), np.arccos(rho * p[2]), rho])
        if rep == 2:
            return pA.copy()
        if rep == 4:
            return np.array([pA[0] / pA[2], pA[1] / pA[2], 1 / pA[2]])
        return np.array([1 / pA[2]])

    def from_lambda(rep, lam, anc, cal, bearing):
        if rep == 0:
            return lam.copy()
        if rep in (1, 3):
            th, ph, rho = lam
            p = np.array([np.cos(th) * np.sin(ph), np.sin(th) * np.sin(ph), np.cos(ph)]) / rho
        elif rep == 2:
            p = lam.copy()
        elif rep == 4:
            p = np.array([lam[0], lam[1], 1.0]) / lam[2]
        else:
            p = bearing / lam[0]
        if rep == 1:
            return p
        R_GtoI, R_ItoC = jpl.quat_2_Rot(anc[:4]), jpl.quat_2_Rot(cal[:4])
        return R_GtoI.T @ R_ItoC.T @ (p - cal[4:]) + anc[4:]

    def perturb_pose(pose, d):  # ov_type::PoseJPL::update: q <- [0.5 dtheta; 1] (x) q, p <- p + dp
        out = pose.copy()
        out[:4] = jpl.quat_left_update(pose[:4], d[:3])
        out[4:] += d[3:]
        return out

    for rep in range(6):
        anc, ancf, cal = rand_pose(), rand_pose(), rand_pose()
        pA = np.array([0.4, -0.3, 3.0]) + 0.2 * rng.normal(size=3)
        pG = jpl.quat_2_Rot(anc[:4]).T @ jpl.quat_2_Rot(cal[:4]).T @ (pA - cal[4:]) + anc[4:] if rep >= 2 else np.array([1.5, -2.0, 4.0])
        pGf = pG + 0.01 * rng.normal(size=3)
        for do_fej in (0, 1):
            g = _rep_call(lib, "ovp_feature_jacobian_representation", rep, do_fej, pG, pGf, pA, anc, ancf, cal)
            o = _rep_call(orc, "orc_feature_jacobian_representation", rep, do_fej, pG, pGf, pA, anc, ancf, cal)
            assert g[3] == o[3] == (1 if rep >= 2 else 0) and g[0].shape == o[0].shape
            assert np.allclose(g[0], o[0], rtol=1e-12, atol=1e-14)
            if rep >= 2:
                assert np.allclose(g[1], o[1], rtol=1e-12, atol=1e-14) and np.allclose(g[2], o[2], rtol=1e-12, atol=1e-14)
        # numerical derivative of p_FinG(lambda, anchor, calib) under the ov_type update rules (no FEJ)
        Hf, Ha, Hc, _ = _rep_call(lib, "ovp_feature_jacobian_representation", rep, 0, pG, pG, pA, anc, anc, cal)
        lam = to_lambda(rep, pG, pA)
        bearing = pA / pA[2]
        f0 = from_lambda(rep, lam, anc, cal, bearing)
        assert np.allclose(f0, pG, atol=1e-12)
        eps = 1e-6
        num = np.zeros((3, len(lam)))
        for k in range(len(lam)):
            d = np.zeros(len(lam))
            d[k] = eps
            num[:, k] = (from_lambda(rep, lam + d, anc, cal, bearing) - from_lambda(rep, lam - d, anc, cal, bearing)) / (2 * eps)
        assert np.allclose(Hf, num, rtol=1e-6, atol=1e-7), (rep, Hf, num)
        if rep >= 2:
            for H, which in ((Ha, 0), (Hc, 1)):
                num = np.zeros((3, 6))
                for k in range(6):
                    d = np.zeros(6)
                    d[k] = eps
                    hi = from_lambda(rep, lam, perturb_pose(anc, d) if which == 0 else anc, perturb_pose(cal, d) if which == 1 else cal, bearing)
                    lo = from_lambda(rep, lam, perturb_pose(anc, -d) if which == 0 else anc, perturb_pose(cal, -d) if which == 1 else cal, bearing)
                    num[:, k] = (hi - lo) / (2 * eps)
                assert np.allclose(H, num, rtol=1e-6, atol=1e-7), (rep, which, H, num)
