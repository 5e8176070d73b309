"""init_vio_plane's orchestration (ov_plane_b200.plane_init_chain) on the CPU oracle: the libstdc++ sort it restates against std::sort itself,
the reference's decisions on a scene with every hazard, and a noise-free room whose planes come out where they were simulated."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import oracle_backend
import oracle_plane_init
from ov_plane_b200 import synth
from ov_plane_b200 import plane_init_chain as pic

SORT_SRC = r"""
#include <algorithm>
#include <cstdio>
#include <vector>
int main() {
  int n;
  while (std::scanf("%d", &n) == 1) {
    std::vector<int> k(n), v(n);
    for (int i = 0; i < n; i++) {
      if (std::scanf("%d", &k[i]) != 1) return 1;
      v[i] = i;
    }
    std::sort(v.begin(), v.end(), [&](int a, int b) { return k[a] < k[b]; });
    for (int i = 0; i < n; i++) std::printf("%d ", v[i]);
    std::printf("\n");
  }
}
"""


def test_sort_model_is_libstdcxx_std_sort(tmp_path):
    """the order of equal track lengths decides RANSAC's draws: the restated introsort must leave ties where g++'s std::sort leaves them"""
    cxx = shutil.which("g++")
    assert cxx, "g++ is needed to build the std::sort reference"
    src, exe = os.path.join(tmp_path, "s.cpp"), os.path.join(tmp_path, "s")
    with open(src, "w") as f:
        f.write(SORT_SRC)
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-o", exe, src])
    rng = np.random.RandomState(0)
    cases = [rng.randint(0, r, size=n) for n in list(range(1, 70)) + [100, 257, 1000] for r in (1, 2, 3, 7, 50)]
    cases += [np.arange(300), np.arange(300)[::-1], np.tile(np.arange(3), 100)]
    out = subprocess.run([exe], input="".join("%d %s\n" % (len(c), " ".join(map(str, c))) for c in cases), capture_output=True, text=True,
                         check=True).stdout.split("\n")
    n_unstable = 0
    for c, line in zip(cases, out):
        mine = pic.libstdcxx_sort(range(len(c)), lambda a, b: c[a] < c[b])
        assert mine == [int(x) for x in line.split()], c
        n_unstable += mine != sorted(range(len(c)), key=lambda i: c[i])
    assert n_unstable > len(cases) // 2  # a stable sort would not do


def _oracle(S, chi2):
    orc = oracle_backend.OracleContext(S.options)
    orc.set_chi2_table(chi2)
    return orc, synth.load_scenario_into(orc, S)


@pytest.mark.parametrize("seed", [0, 2])
def test_reference_decisions_on_the_hazard_scene(seed, chi2_table):
    S, mk = pic.tracks_scene(name="small_planes", seed=seed, px_noise=0.1, keep_in_state=(4,), off_plane=((1, 0.03), (2, 0.045)), ransac_fail_plane=50,
                             n_single=3, n_far=1)
    orc, ch = _oracle(S, chi2_table)
    t = mk(ch)
    n0 = orc.cov_rows()
    r = pic.chain(orc, t, S.options["sigma_constraint"], max_msckf_plane=15)
    fs, pid = r["feat_status"], t["planeid"]
    assert (fs[pid == 0] == 0).all() and (fs[pid == 4] == 0).all()  # no plane / in-state plane: untouched
    assert (fs == -1).sum() == 3 and (fs == -2).any()
    assert list(r["plane_ids"]) == [1, 2, 3, 50]
    st = dict(zip(r["plane_ids"], r["plane_status"]))
    assert st[50] == -2 and st[3] == 1 and -3 in r["plane_status"]
    n_over = 0
    for p, s in r["stages"].items():
        if p != 50:
            assert len(s["grouped"]) == 16  # max_msckf_plane + 1
            cnt = np.diff(t["meas_offset"])
            others = [f for f in np.nonzero((pid == p) & (fs >= 1))[0] if f not in s["grouped"]]
            if others:  # over the cap: the shortest tracks are the ones kept
                n_over += 1
                assert max(cnt[s["grouped"]]) <= min(cnt[others])
    assert n_over >= 2
    consumed = sorted(f for p, s in r["stages"].items() if st[p] == 1 for f in s["refined"])
    assert consumed == sorted(np.nonzero(fs == 1)[0])
    assert orc.cov_rows() == n0 + 3 * sum(v == 1 for v in st.values())
    assert_composition_equals_chain(S, mk, chi2_table)


# (scene, const_init_chi2): plane 1 is noisier than the others, so with a tight const_init_chi2 its initialisation is rejected by the chi2
# test while plane 3, initialised after it at the posterior, passes.  On the oracle plane 1 is accepted from 0.07 up and plane 3 still passes at
# 0.003: 0.01 keeps both decisions a factor of three or more from their thresholds; plane 2 (points +-4.5 cm off its plane) fails the refinement, plane 50 RANSAC
CHI2_SCENE = (dict(name="small_planes", seed=0, px_noise=0.05, keep_in_state=(4,), noisy=((1, 0.3),), off_plane=((2, 0.045),), ransac_fail_plane=50,
                   n_single=3, n_far=1), 0.01)


def assert_composition_equals_chain(S, mk, chi2):
    """the C++ composition on the oracle (real std::sort, tests/oracle_plane_init.cpp) against the Python chain over the oracle's stages"""
    out = []
    for which in ("composed", "chain"):
        orc, ch = _oracle(S, chi2)
        t = mk(ch)
        if which == "composed":
            r = oracle_plane_init.plane_init_tracks(orc, t, S.options["sigma_constraint"], max_msckf_plane=15)
            r["stages"] = oracle_plane_init.stages_of(r, t["planeid"])
        else:
            r = pic.chain(orc, t, S.options["sigma_constraint"], max_msckf_plane=15)
        out.append((r, orc.cov(), [orc.var_get(h) for h in orc.variable_order()]))
    (a, Pa, va), (b, Pb, vb) = out
    for k in ("feat_status", "plane_ids", "plane_status", "new_handles", "cp", "p_FinG"):
        assert np.array_equal(a[k], b[k]), k
    for p in a["plane_ids"]:
        for k in ("grouped", "ransac", "refined"):
            assert a["stages"][int(p)][k] == set(b["stages"][int(p)].get(k, ())), (p, k)
    assert np.array_equal(Pa, Pb) and all(np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) for x, y in zip(va, vb))
    return a


def test_chi2_rejection_then_a_plane_that_initialises(chi2_table):
    kw, c2 = CHI2_SCENE
    S, mk = pic.tracks_scene(**kw)
    S.options["const_init_chi2"] = c2
    r = assert_composition_equals_chain(S, mk, chi2_table)
    st = dict(zip(r["plane_ids"], r["plane_status"]))
    assert st == {1: 0, 2: -3, 3: 1, 50: -2}, st
    assert (r["feat_status"][S.scene_planeid == 1] != 1).all() and (r["feat_status"][S.scene_planeid == 1] == 2).any()  # rejected: nothing consumed


def test_noise_free_room_initialises_its_planes_where_they_are(chi2_table):
    S, mk = pic.tracks_scene(name="small_planes", seed=0, px_noise=0.0)
    orc, ch = _oracle(S, chi2_table)
    r = pic.chain(orc, mk(ch), S.options["sigma_constraint"], max_msckf_plane=100)
    assert (r["plane_status"] == 1).all() and len(r["plane_ids"]) == 4
    for p, cp in zip(r["plane_ids"], r["cp"]):
        err = np.abs(cp - pic.true_plane_cp(int(p))).max()
        assert err < 5e-3, (p, err)  # float32 pixels and the perturbed calibration of the state
        v, _ = orc.var_get(orc.plane_handle(int(p)))
        assert np.abs(v - pic.true_plane_cp(int(p))).max() < 5e-3
