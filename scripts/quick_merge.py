# Device-resident timing of Merge (tg_merge, one GPU) against what a user does without it: tg_sort of the union of the
# inputs.  The inputs are pre-sorted uniform keys; the two are timed alternately with CUDA events after warm-up, the
# TG_K_MERGE kernel time comes from a separate profiled call, and the outputs are compared in the same run (a stable sort of
# the input-major union is exactly the merge).  Prints the card and its power limit with the numbers.
#   python scripts/quick_merge.py [iters]
import ctypes as C
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from thrill_b200 import capi  # noqa: E402

HBM_TBS = 3.35          # H100 SXM data-sheet HBM3 bandwidth (TB/s)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def run_case(c, name, item_bytes, total, k, iters):
    desc = capi.u64_desc() if item_bytes == 8 else capi.kv_key_desc()
    per = [total // k + (1 if j < total % k else 0) for j in range(k)]
    off = np.concatenate([[0], np.cumsum(per)]).astype(np.int64)
    src = c.alloc(total * item_bytes + 64)          # the k sorted inputs back to back (= the input-major union)
    union = c.alloc(total * item_bytes + 64)
    tmp = c.alloc(total * item_bytes + 64)

    def gen(dst, j):
        if item_bytes == 8:
            c.ck(c.L.tg_gen_sort_uniform(c.h, dst, int(off[j]), per[j], 7 + j))
        else:
            c.ck(c.L.tg_gen_reduce_uniform(c.h, dst, int(off[j]), per[j], 7 + j, 1 << 40, 0))
    for j in range(k):
        p = src + int(off[j]) * item_bytes
        gen(p, j)
        c.ck(c.L.tg_radix_sort_local(c.h, C.byref(desc), p, tmp, per[j]))
    c.sync()
    ptrs = (C.c_void_p * k)(*[src + int(off[j]) * item_bytes for j in range(k)])
    sizes = (C.c_size_t * k)(*per)
    in_sum = c.checksum(src, total, item_bytes)

    def merge():
        out, n = C.c_void_p(), C.c_size_t()
        c.ck(c.L.tg_merge(c.h, C.byref(desc), ptrs, sizes, k, C.byref(out), C.byref(n)))
        return out.value, n.value

    def sort():
        out, n = C.c_void_p(), C.c_size_t()
        c.ck(c.L.tg_sort(c.h, C.byref(desc), union, total, 1, C.byref(out), C.byref(n)))
        return out.value, n.value

    def refill_union():
        # tg_sort clobbers its input: the union is copied from the inputs before every sort, untimed (a k = 1 tg_kway_merge
        # is a device-to-device copy)
        c.ck(c.L.tg_kway_merge(c.h, C.byref(desc), src, (C.c_uint64 * 1)(total), 1, union, tmp))
        c.sync()

    t_merge, t_sort = [], []
    for it in range(iters + 2):
        refill_union()
        c.timer_start()
        merge()
        tm = c.timer_stop()
        c.timer_start()
        sout, _ = sort()
        ts = c.timer_stop()
        if it >= 2:
            t_merge.append(tm)
            t_sort.append(ts)
    # outputs of the last round: the merge result (WS_OUT) and the sort result
    mout, mn = merge()
    ok_sorted = c.is_sorted(desc, mout, mn)
    ok_sum = c.checksum(mout, mn, item_bytes) == in_sum
    refill_union()
    sout, sn = sort()
    mout, mn = merge()
    a = c.download(mout, mn * item_bytes)
    b = c.download(sout, sn * item_bytes)
    same = mn == sn == total and np.array_equal(a, b)
    # kernel time of the merge passes
    c.profile_enable(True)
    merge()
    kms, launches = c.profile_get(capi.K_MERGE)
    c.profile_enable(False)
    passes = int(np.ceil(np.log2(k)))
    model = passes * 2 * item_bytes * total            # every pass reads and writes every item once
    mm, ms = float(np.median(t_merge)), float(np.median(t_sort))
    print("%-16s k=%-2d N=%.2e  merge %.3f ms (min %.3f)  sort of the union %.3f ms (min %.3f)  sort/merge %.2fx  | "
          "TG_K_MERGE %.3f ms in %d launches, %d pass(es), %.0f GB/s = %.0f%% of %.2f TB/s (model %d B/item)  | "
          "sorted=%s multiset=%s equal_to_sort=%s"
          % (name, k, total, mm, min(t_merge), ms, min(t_sort), ms / mm, kms, launches, passes, model / kms / 1e6,
             100 * model / kms / 1e6 / (HBM_TBS * 1e3), HBM_TBS, passes * 2 * item_bytes, ok_sorted, ok_sum, same), flush=True)
    for p in (src, union, tmp):
        c.free(p)
    return ok_sorted and ok_sum and same


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    print("card: %s" % card(), flush=True)
    c = capi.Ctx(0)
    ok = True
    for name, ib, total in (("u64", 8, 100000000), ("pair<u64,u64>", 16, 50000000)):
        for k in (2, 4):
            ok = run_case(c, name, ib, total, k, iters) and ok
    c.close()
    print("ALL_OK" if ok else "MISMATCH", flush=True)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
