# Device-resident timing of the Sum / Min / Max actions (tg_all_reduce, one GPU), against what the stock action pays first:
#   u64 sum / min / max     1e8 uint64_t                                    model 8 B/item read
#   f64 sum / min / max     1e8 doubles                                     model 8 B/item read
#   pair max / f64 sum      5e7 pair<uint64_t, V> with ScanSecond<F>        model 16 B/item read
#   fetch                   tg_dev_file_fetch of the same 1e8 x 8 B buffer into page-locked host memory (the D2H a GPU node
#                           makes before a stock action can fold anything)
# Calls are timed with CUDA events after warm-up (median and min); the per-kernel times come from a separate profiled call
# (TG_K_SCAN launches in order: tile reduce, fold), with the achieved bytes/s at the model's bytes.  Each result is checked
# against the numpy model (tests/action_ref.py): bit for bit, double sums within 1e-9 relative.  Prints the card and its power
# limit.
#   python scripts/quick_action.py [iters]
import ctypes as C
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from thrill_b200 import capi  # noqa: E402
import action_ref as A  # noqa: E402
import scan_ref as S  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
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


def run_case(c, name, arr, op, pair, iters):
    n, ib = len(arr), 16 if pair else 8
    d = c.to_device(arr)
    out = np.zeros(2, np.uint64)
    desc = capi.ScanDesc(ib, op)

    def call():
        c.ck(c.L.tg_all_reduce(c.h, C.byref(desc), d, n, None, out.ctypes.data))
    med, best = timed(c, call, iters)
    c.profile_enable(True)
    call()
    per = c.profile_list(capi.K_SCAN)
    c.profile_enable(False)
    got = (int(out[0]), int(out[1])) if pair else (0, int(out[0]))
    want = A.all_reduce([arr], op, pair)
    if op == A.OP_SUM_F64:
        g, w = A._f(got[1]), A._f(want[1])
        ok = got[0] == want[0] and abs(g - w) <= 1e-9 * max(1.0, abs(w))
    else:
        ok = got == want
    print("%-9s n=%.0e  %.3f ms (min %.3f) = %.2f TB/s at the model's %d B/item; reduce %.3f ms = %.2f TB/s, fold %.3f ms; %s"
          % (name, n, med, best, n * ib / best / 1e9, ib, per[0], n * ib / per[0] / 1e9, per[1],
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
    for name, op in (("u64 sum", A.OP_SUM_U64), ("u64 min", A.OP_MIN_U64), ("u64 max", A.OP_MAX_U64)):
        ok = run_case(c, name, x, op, False, iters) and ok
    f = S.f64_words(rng.standard_normal(n))
    for name, op in (("f64 sum", A.OP_SUM_F64), ("f64 min", A.OP_MIN_F64), ("f64 max", A.OP_MAX_F64)):
        ok = run_case(c, name, f, op, False, iters) and ok
    del f
    pairs = S.pairs(x[:n // 2], x[n // 2:] >> np.uint64(12))
    ok = run_case(c, "pair max", pairs, A.OP_MAX_U64, True, iters) and ok
    pairs["val"] = S.f64_words(rng.standard_normal(n // 2))
    ok = run_case(c, "pair fsum", pairs, A.OP_SUM_F64, True, iters) and ok
    del pairs
    # what the stock action pays first: the device File fetched to the host
    d = c.to_device(x)
    f = capi.DevFile(d, n, 8, 0)
    host = c.host_alloc(n * 8)
    blk = (capi.Block * 1)()
    blk[0].data, blk[0].bytes = host.ctypes.data, n * 8

    def fetch():
        c.ck(c.L.tg_dev_file_fetch(c.h, C.byref(f), blk, 1))
    med, best = timed(c, fetch, max(3, iters // 2))
    ok = ok and np.array_equal(host.view(np.uint64), x)
    print("%-9s n=%.0e  %.3f ms (min %.3f) = %.1f GB/s D2H into page-locked memory" % ("fetch", n, med, best, n * 8 / best / 1e6),
          flush=True)
    c.host_free(host)
    c.free(d)
    c.close()
    print("ALL_OK" if ok else "MISMATCH", flush=True)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
