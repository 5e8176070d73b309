"""Timeline of the fused Cholesky kernel (cholfused.cu) on a synthetic SPD system: per-CTA globaltimer stamps."""
import ctypes as C, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from ov_plane_b200 import api, synth

n = int(sys.argv[1]) if len(sys.argv) > 1 else 474
mrows = int(sys.argv[2]) if len(sys.argv) > 2 else 512
S = synth.make_scenario("tiny_points")
ctx = api.Context(S.options, device=0, max_state=576, max_meas_rows=4096, debug=True)
for (nn, mm) in ((n, 0), (n, mrows), (128, 0), (64, 0)):
    T = (nn + 63) // 64
    cap = 3 + 16 * (T * (T + 1) // 2 + 40) + 64
    out = np.zeros(cap)
    ctx._ck(ctx.lib.ovp_debug_chol_fused(ctx.h, nn, mm, 50, out.ctypes.data_as(C.c_void_p), cap))
    print("n=%d mrows=%d: fused chol %.1f us (fill+factor %.1f, fill %.1f)" % (nn, mm, out[0] - out[1], out[0], out[1]))
    ncta = int(out[2])
    ts = out[3:3 + 16 * ncta].reshape(ncta, 16) / 1e3  # us
    def bidx(i, j):
        return sum(T - q for q in range(j)) + (i - j)
    if nn == n:
        sp = ts[0]
        print("  spine: start %.1f" % sp[0])
        for k in range(min(3, T)):
            s0, s1 = sp[1 + 2 * k], sp[2 + 2 * k]
            nxt = sp[3 + 2 * k] if k + 1 < min(3, T) else float("nan")
            print("  k=%d potrf %6.1f -> %6.1f (%.1f us)   until next potrf (trinv, publish, panel, update): %.1f us" % (k, s0, s1, s1 - s0, nxt - s1))
        print("  last CTA end %.1f us" % ts[:, 15].max())
        # producer path of the tiles the spine needs for step k+1 (us, same clock as the spine's stamps)
        for k in range(1, min(4, T - 1)):
            pan = ts[bidx(k + 1, k - 1)]
            us, ud = ts[bidx(k + 1, k)], ts[bidx(k + 1, k + 1)] if k + 1 < T else None
            print("  step %d: spine potrf %.1f..%.1f | tile(%d,%d) Linv loaded %.1f solved %.1f published %.1f | tile(%d,%d) updated %.1f published %.1f | tile(%d,%d) updated %.1f published %.1f"
                  % (k, sp[1 + 2 * k] if k < 3 else float("nan"), sp[2 + 2 * k] if k < 3 else float("nan"), k + 1, k - 1, pan[5], pan[6], pan[7], k + 1, k, us[3], us[4], k + 1, k + 1, ud[3], ud[4]))
        ph = out[3 + 16 * ncta:3 + 16 * ncta + 29]
        ls = out[3 + 16 * ncta + 30:3 + 16 * ncta + 54]
        names = ["potrf start"] + [x for b in range(4) for x in ("chain%d" % b, "sync%d" % b, "trail%d+sync" % b)] + ["trinv zero", "trinv base16", "merge16 T", "merge16 X", "merge32 T", "merge32 X",
                 "store Linv", "signal D", "store L", "(unused)", "cp.async wait", "sync", "panel mma", "store panel", "signal P", "update mma"]
        prev = 0.0
        line = []
        for nm, v in zip(names, ph):
            if v >= 0:
                line.append("%s %d" % (nm, v - prev))
                prev = v
        print("  spine k=1 phase cycles: " + " | ".join(line))
        print("  pivot loop of panel p starts (cycles since potrf start): " + " ".join("%d" % v for v in ls[:4]) + "  potrf entry %d, after its first barrier %d; chain warps reach the named barrier of panel 0 at %s, of panel 1 at %s" % (ls[4], ls[5], " ".join("%d" % v for v in ls[10:14]), " ".join("%d" % v for v in ls[14:18])) + "; panel 0 set-up: branch entry %d, rows loaded %d, diagonal shuffled %d" % (ls[20], ls[21], ls[22]) + "   (chain p ends at " + " ".join("%d" % ph[1 + 3 * b] for b in range(4)) + ")")
        if mm:
            print("  row-block CTAs end: min %.1f max %.1f" % (ts[T * (T + 1) // 2:, 15].min(), ts[T * (T + 1) // 2:, 15].max()))

# Paired launch of a compressed update (chol_fused_pair): per step k, when the Gram spine released D(k) and when the innovation spine
# started step k, and the lag in Gram steps.  Systems of the benchmark's shapes: a plane update (474 columns with z, 470 pivots) and the
# point update (471, 470), 512 rows of M.
def _p(x):
    return x.ctypes.data_as(C.c_void_p)


for tag, nc, npiv in (("plane", 473, 470), ("point", 470, 470)):
    N = 512
    rng = np.random.default_rng(nc)
    H = rng.standard_normal((nc + 24, nc + 1))
    G = np.asfortranarray(np.tril(H.T @ H))
    A = rng.standard_normal((N, N))
    P = np.asfortranarray(A @ A.T / N + np.eye(N))
    cols = np.ascontiguousarray(np.sort(rng.choice(N, size=nc, replace=False)), dtype=np.int32)
    L, M, Y = np.zeros((nc + 1, npiv), order="F"), np.zeros((N, npiv), order="F"), np.zeros((N, npiv), order="F")
    LS, w, tl = np.zeros((npiv, npiv), order="F"), np.zeros(npiv), np.zeros(64)
    chi2, gate, info = C.c_double(0.0), C.c_int(0), np.zeros(1, dtype=np.int32)
    for _ in range(3):  # the last run's stamps
        ctx._ck(ctx.lib.ovp_debug_chol_pair(ctx.h, _p(G), nc, npiv, C.c_double(1e-11), _p(P), N, _p(cols), C.c_double(-1.0), _p(L), _p(M), _p(LS),
                                            _p(Y), _p(w), C.byref(chi2), C.byref(gate), _p(info), _p(tl)))
    if not info[0]:
        print("%s: the pair does not fit one launch on this device" % tag)
        continue
    Tp = (npiv + 63) // 64
    d, s = tl[:Tp], tl[32:32 + Tp]
    step = (d[-1] - d[0]) / max(1, Tp - 1)  # mean Gram spine step
    print("%s update (nc=%d, npiv=%d, N=%d), pair, us from the first stamp; Gram step %.1f us" % (tag, nc, npiv, N, step))
    for k in range(Tp):
        print("  k=%d  Gram spine released D(k) %7.1f   innovation spine started step k %7.1f   lag %.2f Gram steps" % (k, d[k], s[k], (s[k] - d[k]) / step))
