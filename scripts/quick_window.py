# Device-resident timing of Window (tg_window, one GPU), against what the stock node pays first:
#   u64 sum / max       1e8 uint64_t at k = 2, 64 and 4096, overlapping and disjoint
#   f64 sum             1e8 doubles, k = 64, overlapping and disjoint
#   pair fsum / max     5e7 pair<uint64_t, V> with ScanSecond<F>, k = 64
#   fetch               tg_dev_file_fetch of the same 1e8 x 8 B buffer into page-locked host memory (the D2H the stock node
#                       needs before it folds anything)
# Calls are timed with CUDA events after warm-up (median of `iters`, and min); the kernel time comes from a separate profiled
# call (TG_K_WINDOW), with TB/s at the algorithmic bytes: (1 + 1/m) s read per item for m = max(1, 4096 / k) blocks per CTA (s for
# disjoint windows, which need no next block), s written per output.  Results are checked against the model in the same run:
# integer sums exactly (prefix sums mod 2^64), double sums against tests/window_ref.emulate_sum on a prefix, maxima at sampled
# windows.  Prints the card, its power limit and SM clock.
#   python scripts/quick_window.py [iters]
import ctypes as C
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from thrill_b200 import capi  # noqa: E402
import scan_ref as S  # noqa: E402
import window_ref as W  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def timed(c, call, iters):
    times = []
    for it in range(iters + 2):
        c.timer_start()
        call()
        t = c.timer_stop()
        if it >= 2:
            times.append(t)
    return float(np.median(times)), min(times)


def check(vals, got, op, k, form, first=None, pair_first=None):
    """sums of integers in full; otherwise sampled windows of the model / the emulated bracketing"""
    n = len(vals)
    s, ln = W.runs(n, k, form)
    if len(got) != len(s):
        return False
    if op == W.OP_SUM_U64:
        cs = np.concatenate([[np.uint64(0)], np.cumsum(vals, dtype=np.uint64)])
        return np.array_equal(got, cs[s + ln] - cs[s])
    rng = np.random.RandomState(k)
    idx = np.unique(np.concatenate([rng.randint(0, len(s), 3000), [0, len(s) - 1]]))
    if op == W.OP_SUM_F64:
        m = min(n, 300_000)
        ms = len(W.runs(m, k, form)[0]) - (k - 1 if form == W.PARTIAL else 1 if form == W.DISJOINT and m % k else 0)
        return np.array_equal(W.emulate_sum(vals[:m], k, form)[:ms], got[:ms])
    want = W.fold_runs(vals, op, s[idx], ln[idx])
    return np.array_equal(want, got[idx])


def run_case(c, name, vals, op, k, form, iters, firsts=None):
    pair = firsts is not None
    n, ib = len(vals), 16 if pair else 8
    arr = np.stack([firsts, vals], axis=1) if pair else vals
    d = c.to_device(arr)
    desc = capi.ScanDesc(ib, op)
    out, m = C.c_void_p(), C.c_size_t()

    def call():
        c.ck(c.L.tg_window(c.h, C.byref(desc), d, n, k, form, C.byref(out), C.byref(m)))
    med, best = timed(c, call, iters)
    c.profile_enable(True)
    call()
    kern = c.profile_list(capi.K_WINDOW)
    c.profile_enable(False)
    raw = c.download(out.value, m.value * ib).view(np.uint64)
    got = raw.reshape(-1, 2)[:, 1] if pair else raw
    ok = check(vals, got, op, k, form)
    if pair:
        s, ln = W.runs(n, k, form)
        ok = ok and np.array_equal(raw.reshape(-1, 2)[:, 0], firsts[s + ln - 1])
    # a CTA stages its m blocks and, for overlapping windows, the next one
    restage = 0.0 if form == W.DISJOINT else 1.0 / max(1, 4096 // k)
    model = n * ib * (1 + restage) + m.value * ib
    print("%-10s k=%-4d %-8s n=%.0e  %.3f ms (min %.3f); kernel %.3f ms = %.2f TB/s at %.1f B/item; %s"
          % (name, k, W.FORMS[form], n, med, best, kern[0], model / kern[0] / 1e9, model / n,
             "equal to the model" if ok else "DIFFERENT from the model"), flush=True)
    c.free(d)
    return ok


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    print("card: %s" % card(), flush=True)
    n = 100_000_000
    rng = np.random.default_rng(5)
    c = capi.Ctx(0)
    x = rng.integers(0, 1 << 62, n, dtype=np.uint64)
    ok = True
    for k in (2, 64, 4096):
        for form in (W.FULL, W.DISJOINT):
            for name, op in (("u64 sum", W.OP_SUM_U64), ("u64 max", W.OP_MAX_U64)):
                ok = run_case(c, name, x, op, k, form, iters) and ok
    f = S.f64_words(rng.standard_normal(n))
    for form in (W.FULL, W.DISJOINT):
        ok = run_case(c, "f64 sum", f, W.OP_SUM_F64, 64, form, iters) and ok
    del f
    h = n // 2
    ok = run_case(c, "pair max", x[h:] >> np.uint64(12), W.OP_MAX_U64, 64, W.FULL, iters, firsts=x[:h]) and ok
    ok = run_case(c, "pair fsum", S.f64_words(rng.standard_normal(h)), W.OP_SUM_F64, 64, W.FULL, iters, firsts=x[:h]) and ok
    d = c.to_device(x)
    f = capi.DevFile(d, n, 8, 0)
    host = c.host_alloc(n * 8)
    blk = (capi.Block * 1)()
    blk[0].data, blk[0].bytes = host.ctypes.data, n * 8

    def fetch():
        c.ck(c.L.tg_dev_file_fetch(c.h, C.byref(f), blk, 1))
    med, best = timed(c, fetch, max(3, iters // 2))
    ok = ok and np.array_equal(host.view(np.uint64), x)
    print("%-10s n=%.0e  %.3f ms (min %.3f) = %.1f GB/s D2H into page-locked memory" % ("fetch", n, med, best, n * 8 / best / 1e6),
          flush=True)
    c.host_free(host)
    c.free(d)
    c.close()
    print("card: %s" % card(), flush=True)
    print("ALL_OK" if ok else "MISMATCH", flush=True)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
