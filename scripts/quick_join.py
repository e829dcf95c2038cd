# Device-resident timing of InnerJoin (tg_inner_join, one GPU) on two shapes:
#   foreign key: 1e8 left pairs with keys uniform over 2^26 against the 2^26 distinct right keys (1e8 outputs)
#   uniform:     1e8 x 1e8 pairs with keys uniform over 2^27 (about 7.5e7 outputs)
# Calls are timed with CUDA events after warm-up; the TG_K_JOIN launches (count splits, count, tile scan, offsets, emit splits,
# emit) come from a separate profiled call, with their achieved bytes/s against the data-sheet HBM bandwidth.  The output of
# the same run is checked against the numpy model (tests/join_ref.py) by tg_checksum of both.  Prints the card and its power
# limit with the numbers.
#   python scripts/quick_join.py [iters]
import ctypes as C
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from thrill_b200 import capi  # noqa: E402
import join_ref as J  # noqa: E402

HBM_TBS = 3.35          # H100 SXM data-sheet HBM3 bandwidth (TB/s)
KERNELS = ["count splits", "count", "tile scan", "offsets", "emit splits", "emit"]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def run_case(c, name, left, right, fn, iters):
    nl, nr = len(left), len(right)
    s_out = J.out_dtype(fn).itemsize
    dl, dr = c.to_device(left), c.to_device(right)
    desc = capi.JoinDesc(16, fn)

    def join():
        out, n = C.c_void_p(), C.c_size_t()
        c.ck(c.L.tg_inner_join(c.h, C.byref(desc), dl, nl, dr, nr, C.byref(out), C.byref(n)))
        return out.value, n.value

    times = []
    for it in range(iters + 2):
        c.timer_start()
        join()
        t = c.timer_stop()
        if it >= 2:
            times.append(t)
    c.profile_enable(True)
    out, m = join()
    per = c.profile_list(capi.K_JOIN)
    part_ms, _ = c.profile_get(capi.K_PARTITION)
    hist_ms, _ = c.profile_get(capi.K_RADIX_HIST)
    fix_ms, _ = c.profile_get(capi.K_FIXUP)
    c.profile_enable(False)
    got = c.checksum(out, m, s_out)
    ref = J.join_local(left, right, fn)
    dref = c.to_device(ref)
    ok = len(ref) == m and c.checksum(dref, m, s_out) == got
    c.free(dref)
    # bytes each kernel needs (DESIGN.md §5): count reads both sides and writes 8 B per left item; the offsets pass reads and
    # writes 8 B per left item; the emit writes the outputs and reads the right item of every output, the left item and its
    # offset and counts once
    model = {"count": 16 * (nl + nr) + 8 * nl, "offsets": 16 * nl, "emit": s_out * m + 16 * m + 32 * nl}
    print("%-12s nl=%.2e nr=%.2e m=%.3e  tg_inner_join %.3f ms (min %.3f)  | sorts: partition %.3f ms, hist %.3f ms, fixup %.3f ms"
          % (name, nl, nr, m, float(np.median(times)), min(times), part_ms, hist_ms, fix_ms), flush=True)
    for k, ms in zip(KERNELS, per):
        extra = ""
        if k in model:
            extra = "  %.0f GB/s = %.0f%% of %.2f TB/s" % (model[k] / ms / 1e6, 100 * model[k] / ms / 1e6 / (HBM_TBS * 1e3), HBM_TBS)
        print("    TG_K_JOIN %-12s %.3f ms%s" % (k, ms, extra), flush=True)
    print("    checksum vs model: %s" % ("equal" if ok else "DIFFERENT"), flush=True)
    c.free(dl)
    c.free(dr)
    return ok


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    print("card: %s" % card(), flush=True)
    rng = np.random.default_rng(5)
    n = 100_000_000
    c = capi.Ctx(0)
    ok = True
    left = np.empty(n, J.KV)
    left["key"] = rng.integers(0, 1 << 26, n, dtype=np.uint64)
    left["val"] = np.arange(n, dtype=np.uint64)
    right = np.empty(1 << 26, J.KV)
    right["key"] = rng.permutation(1 << 26).astype(np.uint64)
    right["val"] = rng.integers(0, 1 << 63, 1 << 26, dtype=np.uint64)
    ok = run_case(c, "foreign key", left, right, J.KEY_VALUES, iters) and ok
    right = np.empty(n, J.KV)
    left["key"] = rng.integers(0, 1 << 27, n, dtype=np.uint64)
    right["key"] = rng.integers(0, 1 << 27, n, dtype=np.uint64)
    right["val"] = rng.integers(0, 1 << 63, n, dtype=np.uint64)
    ok = run_case(c, "uniform", left, right, J.KEY_VALUES, iters) and ok
    c.close()
    print("ALL_OK" if ok else "MISMATCH", flush=True)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
