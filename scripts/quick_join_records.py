# Device-resident timing of InnerJoin on records (tg_inner_join_records, one GPU), against the pair join and against what the
# stock JoinNode pays first:
#   tpch      6e7 x 176-byte line items ⋈ 1.5e7 x 152-byte orders, key = an 8-byte orderkey at offset 0, every line item
#             matching one order (a foreign-key join): 6e7 x 328-byte outputs, 19.7 GB
#   uniform   6e7 x 176 B ⋈ 6e7 x 152 B, keys uniform over 6e7 on both sides (about 6e7 outputs, many-to-many)
#   pairs     1e8 16-byte pairs ⋈ 2^26 pairs with distinct keys, through the record path (32-byte outputs) and through the
#             existing pair join (JoinKeyValues, 24-byte outputs)
#   fetch     tg_dev_file_fetch of both TPC-H inputs into page-locked host memory (the D2H the stock JoinNode needs first)
# Calls are timed with CUDA events after warm-up (median of `iters`, and min).  One profiled call per case splits the kernels
# into tuples + sorts (TG_K_OTHER and the radix sort's classes), count + scan (the first four TG_K_JOIN launches) and emit (the
# last two).  The emit's bytes/s are at its model: (s_L + s_R) read + (s_L + s_R) written per output, 16 per output for the
# positions, 32 per left item.  Every output is checked in the same run against a model built on the device with torch: the
# order-independent checksum (tg_checksum) of the whole output and 200 sampled rows.  Prints the card, its power limit and SM clock.
#   python scripts/quick_join_records.py [iters]
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
from thrill_b200 import capi  # noqa: E402

DEV = torch.device("cuda", 0)
SORT_CLASSES = (capi.K_OTHER, capi.K_RADIX_HIST, capi.K_PARTITION, capi.K_MERGE, capi.K_FIXUP, capi.K_SEGCOUNT)


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


def records(n, s, keys, g):
    """n records of s bytes (int32 words of random bits) with the 8-byte key at offset 0"""
    r = torch.randint(-(1 << 31), 1 << 31, (n, s // 4), dtype=torch.int32, device=DEV, generator=g)
    r.view(torch.int64)[:, 0] = keys
    return r


def model_rows(left, right, lkey, rkey, out_words):
    """the one-worker result on the device: (key, left position, right position) order, left record then right record"""
    ol = torch.sort(lkey, stable=True).indices
    orr = torch.sort(rkey, stable=True).indices
    KL, KR = lkey[ol], rkey[orr]
    lo = torch.searchsorted(KR, KL, right=False)
    cnt = torch.searchsorted(KR, KL, right=True) - lo
    m = int(cnt.sum())
    ref = torch.empty((m, out_words), dtype=torch.int32, device=DEV)
    off = torch.cumsum(cnt, 0) - cnt
    lw = left.shape[1]
    step = 1 << 22
    for a in range(0, len(KL), step):                    # left items [a, a + step) and their outputs
        c = cnt[a:a + step]
        li = torch.repeat_interleave(torch.arange(a, a + len(c), device=DEV), c)
        if not len(li):
            continue
        j0 = int(off[a])
        j = torch.arange(j0, j0 + len(li), device=DEV)
        ri = lo[li] + (j - off[li])
        ref[j0:j0 + len(li), :lw] = left[ol[li]]
        ref[j0:j0 + len(li), lw:] = right[orr[ri]]
    return ref, m


def run_case(c, name, left, right, lkey, rkey, iters, model=True):
    nl, nr = left.shape[0], right.shape[0]
    lb, rb = left.shape[1] * 4, right.shape[1] * 4
    d = capi.JoinRecordsDesc(lb, rb, 0, 8, 0, 8)
    out, m = C.c_void_p(), C.c_size_t()

    def call():
        c.ck(c.L.tg_inner_join_records(c.h, C.byref(d), left.data_ptr(), nl, right.data_ptr(), nr, C.byref(out), C.byref(m)))
    torch.cuda.synchronize()
    med, best = timed(c, call, iters)
    c.profile_enable(True)
    call()
    join = c.profile_list(capi.K_JOIN)
    sort = sum(c.profile_get(k)[0] for k in SORT_CLASSES)
    c.profile_enable(False)
    count, emit = sum(join[:4]), sum(join[4:])
    mm = m.value
    emit_bytes = mm * (2 * (lb + rb) + 16) + 32 * nl
    ok = True
    if model:
        got = c.checksum(out.value, mm, lb + rb)
        ref, m_ref = model_rows(left, right, lkey, rkey, (lb + rb) // 4)
        torch.cuda.synchronize()
        ok = m_ref == mm and c.checksum(ref.data_ptr(), mm, lb + rb) == got
        rng = np.random.default_rng(1)
        for j in np.concatenate([[0, mm - 1], rng.integers(0, mm, 198)]) if mm else []:
            row = c.download(out.value + int(j) * (lb + rb), lb + rb)
            ok = ok and np.array_equal(row, ref[int(j)].cpu().numpy().view(np.uint8))
        del ref
        torch.cuda.empty_cache()
    print("%-9s %.1e x %d B ⋈ %.1e x %d B -> %.3e x %d B: %.2f ms (min %.2f); kernels: tuples + sorts %.2f, count + scan %.2f, "
          "emit %.2f ms (%.0f MB at the model, %.2f TB/s); %s"
          % (name, nl, lb, nr, rb, mm, lb + rb, med, best, sort, count, emit, emit_bytes / 1e6,
             emit_bytes / emit / 1e9 if emit > 0 else 0.0, "equal to the model" if ok else "DIFFERENT from the model"), flush=True)
    return ok, out.value, mm


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    print("card: %s" % card(), flush=True)
    c = capi.Ctx(0)
    g = torch.Generator(device=DEV).manual_seed(5)
    ok = True
    # TPC-H-shaped foreign-key join
    nl, nr = 60_000_000, 15_000_000
    rkey = torch.randperm(nr, device=DEV, generator=g)
    lkey = torch.randint(0, nr, (nl,), device=DEV, generator=g)
    left, right = records(nl, 176, lkey, g), records(nr, 152, rkey, g)
    ok = run_case(c, "tpch", left, right, lkey, rkey, iters)[0] and ok
    # what the stock node pays first: both inputs to the host
    host = c.host_alloc(nl * 176 + nr * 152)
    files = [capi.DevFile(left.data_ptr(), nl, 176, 0), capi.DevFile(right.data_ptr(), nr, 152, 0)]
    blks = [(capi.Block * 1)(), (capi.Block * 1)()]
    blks[0][0].data, blks[0][0].bytes = host.ctypes.data, nl * 176
    blks[1][0].data, blks[1][0].bytes = host.ctypes.data + nl * 176, nr * 152

    def fetch():
        for f, b in zip(files, blks):
            c.ck(c.L.tg_dev_file_fetch(c.h, C.byref(f), b, 1))
    med, best = timed(c, fetch, max(3, iters // 2))
    fb = nl * 176 + nr * 152
    print("%-9s %.1f GB: %.2f ms (min %.2f) = %.1f GB/s D2H into page-locked memory" % ("fetch", fb / 1e9, med, best, fb / best / 1e6),
          flush=True)
    c.host_free(host)
    del left, right, lkey, rkey
    torch.cuda.empty_cache()
    # uniform keys on both sides
    n = 60_000_000
    lkey = torch.randint(0, n, (n,), device=DEV, generator=g)
    rkey = torch.randint(0, n, (n,), device=DEV, generator=g)
    left, right = records(n, 176, lkey, g), records(n, 152, rkey, g)
    ok = run_case(c, "uniform", left, right, lkey, rkey, iters)[0] and ok
    del left, right, lkey, rkey
    torch.cuda.empty_cache()
    # 16-byte pairs: the record path against the pair join
    n, u = 100_000_000, 1 << 26
    rkey = torch.randperm(u, device=DEV, generator=g)
    lkey = torch.randint(0, u, (n,), device=DEV, generator=g)
    left, right = records(n, 16, lkey, g), records(u, 16, rkey, g)
    r_ok, rec_out, m_rec = run_case(c, "pairs", left, right, lkey, rkey, iters)
    ok = r_ok and ok
    # the record path's rows (k, v1, k, v2) re-laid out as (k, v1, v2), out of the ctx-owned workspace before the pair join runs
    c.sync()
    rec = device_view(rec_out, (m_rec, 8))
    kvv = torch.cat([rec[:, :4], rec[:, 6:]], dim=1).contiguous()
    del rec
    out, m = C.c_void_p(), C.c_size_t()
    d = capi.JoinDesc(16, capi.JOIN_KEY_VALUES)

    def pair_call():
        c.ck(c.L.tg_inner_join(c.h, C.byref(d), left.data_ptr(), n, right.data_ptr(), u, C.byref(out), C.byref(m)))
    med, best = timed(c, pair_call, iters)
    c.profile_enable(True)
    pair_call()
    join = c.profile_list(capi.K_JOIN)
    sort = sum(c.profile_get(k)[0] for k in SORT_CLASSES)
    c.profile_enable(False)
    same = m.value == m_rec and c.checksum(out.value, m.value, 24) == c.checksum(kvv.data_ptr(), m_rec, 24)
    ok = ok and same
    print("%-9s %.1e x 16 B ⋈ %.1e x 16 B -> %.3e x 24 B (JoinKeyValues): %.2f ms (min %.2f); kernels: sorts %.2f, count + scan "
          "%.2f, emit %.2f ms; %s" % ("pair_join", n, u, m.value, med, best, sort, sum(join[:4]), sum(join[4:]),
                                      "rows equal to the record path's" if same else "DIFFERENT from the record path"), flush=True)
    c.close()
    print("card: %s" % card(), flush=True)
    print("ALL_OK" if ok else "MISMATCH", flush=True)
    return 0 if ok else 1


class _DevArray(object):
    """a raw device pointer as a torch-readable array (__cuda_array_interface__): no copy"""

    def __init__(self, ptr, shape):
        self.__cuda_array_interface__ = {"data": (ptr, False), "shape": shape, "typestr": "<i4", "version": 2}


def device_view(ptr, shape):
    return torch.as_tensor(_DevArray(ptr, shape), device=DEV)


if __name__ == "__main__":
    sys.exit(main())
