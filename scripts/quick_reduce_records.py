# Device-resident timing of ReduceByKey on records (tg_reduce_by_key_records, one GPU), against the pair reduce and against what
# the stock ReduceNode pays first:
#   kmeans16 / kmeans1024  1e8 x 40-byte ClosestCentroid records {u64 cluster_id; double p[3]; u64 count}, key = cluster_id
#                          uniform over 16 or 1024 keys, runs {8, 3, SUM_F64}, {32, 1, SUM_U64}
#   tpch                   6e7 x 176-byte line items, a 1-byte key at offset 0 uniform over 4 keys, four runs: quantity
#                          (SUM_U64), extendedprice, discount, tax (SUM_F64)
#   manykeys               1e8 x 32-byte records, keys uniform over 2^26, runs {8, 2, SUM_F64}, {24, 1, SUM_U64}
#   pairs                  1e8 16-byte pairs, keys uniform over 2^26, SUM_U64: through the record path and through tg_reduce_by_key
#   fetch                  tg_dev_file_fetch of the kmeans input into page-locked host memory (the D2H the stock node needs first)
# Doubles are integers of magnitude < 2^20, so every bracketing gives the exact sum.  Calls are timed with CUDA events after
# warm-up (median of `iters`, and min).  One profiled call per case splits the kernels into tuples + sort (TG_K_OTHER and the radix
# sort's classes) and the four TG_K_REDUCE_RECORDS launches (head count, tile scan, segmented reduce, cut groups).  The segmented
# reduce's bytes/s are at its model: 16 B of tuple + the run words read per item, m * s written.  Every output is checked in the
# same run against a model built on the device with torch (stable sort, first record per key, index_add of the fields): the
# count and the order-independent checksum (tg_checksum) of the whole output.  Prints the card, its power limit and SM clock.
#   python scripts/quick_reduce_records.py [iters]
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


def records(n, s, key_bytes, universe, runs, g):
    """n records of s bytes (random int32 words), the key (uniform over universe) at offset 0, run fields set: doubles are integers
    of magnitude < 2^20, integers below 2^20"""
    r = torch.randint(-(1 << 31), 1 << 31, (n, s // 4), dtype=torch.int32, device=DEV, generator=g)
    keys = torch.randint(0, universe, (n,), dtype=torch.int64, device=DEV, generator=g)
    b = r.view(torch.uint8)
    kb = keys.view(torch.uint8).view(n, 8)
    b[:, :key_bytes] = kb[:, :key_bytes]
    if key_bytes < 8:
        b[:, key_bytes:8] = 0                      # (the model's key is the first 8 bytes)
    w = r.view(torch.int64) if s % 8 == 0 else None
    for off, cnt, op in runs:
        v = torch.randint(-(1 << 20), 1 << 20, (n, cnt), dtype=torch.int64, device=DEV, generator=g)
        w[:, off // 8:off // 8 + cnt] = v.double().view(torch.int64) if op == capi.OP_SUM_F64 else v.abs()
    return r, keys


def model_checksum(c, r, runs):
    """the one-worker result on the device: rows of the first record per key, run fields summed; (m, checksum)"""
    w = r.view(torch.int64)
    k = w[:, 0]
    srt = torch.sort(k, stable=True)
    ks, order = srt.values, srt.indices
    head = torch.ones(len(ks), dtype=torch.bool, device=DEV)
    head[1:] = ks[1:] != ks[:-1]
    gid = torch.cumsum(head.to(torch.int64), 0) - 1
    m = int(gid[-1]) + 1 if len(gid) else 0
    out = w[order[head]].clone()
    for off, cnt, op in runs:
        f = w[order, off // 8:off // 8 + cnt]
        if op == capi.OP_SUM_F64:
            acc = torch.zeros((m, cnt), dtype=torch.float64, device=DEV).index_add_(0, gid, f.view(torch.float64))
            out[:, off // 8:off // 8 + cnt] = acc.view(torch.int64)
        else:
            out[:, off // 8:off // 8 + cnt] = torch.zeros((m, cnt), dtype=torch.int64, device=DEV).index_add_(0, gid, f)
    torch.cuda.synchronize()
    return m, c.checksum(out.data_ptr(), m, r.shape[1] * 4)


def run_case(c, name, r, key_bytes, runs, iters):
    n, s = r.shape[0], r.shape[1] * 4
    d = capi.reduce_records_desc(s, 0, key_bytes, runs)
    out, m = C.c_void_p(), C.c_size_t()

    def call():
        c.ck(c.L.tg_reduce_by_key_records(c.h, C.byref(d), r.data_ptr(), n, C.byref(out), C.byref(m)))
    torch.cuda.synchronize()
    med, best = timed(c, call, iters)
    c.profile_enable(True)
    call()
    rr = c.profile_list(capi.K_REDUCE_RECORDS)
    sort = sum(c.profile_get(k)[0] for k in SORT_CLASSES)
    c.profile_enable(False)
    heads, scan, red = rr[0], rr[1], rr[2]
    cut = rr[3] if len(rr) > 3 else 0.0
    nf = sum(cnt for _, cnt, _ in runs)
    mm = m.value
    red_bytes = n * (16 + 8 * nf) + mm * s
    got = c.checksum(out.value, mm, s)
    m_ref, want = model_checksum(c, r, runs)
    ok = m_ref == mm and want == got
    print("%-10s %.1e x %d B, %d fields -> %d keys: %.2f ms (min %.2f); kernels: tuples + sort %.2f, heads %.3f, scan %.3f, "
          "reduce %.3f (%.0f MB at the model, %.2f TB/s), cut %.3f ms; %s"
          % (name, n, s, nf, mm, med, best, sort, heads, scan, red, red_bytes / 1e6, red_bytes / red / 1e9 if red > 0 else 0.0,
             cut, "equal to the model" if ok else "DIFFERENT from the model"), flush=True)
    torch.cuda.empty_cache()
    return ok


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    print("card:", card(), flush=True)
    c = capi.Ctx(0)
    g = torch.Generator(device=DEV)
    g.manual_seed(1)
    ok = True
    km = [(8, 3, capi.OP_SUM_F64), (32, 1, capi.OP_SUM_U64)]
    for universe in (16, 1024):
        r, _ = records(100_000_000, 40, 8, universe, km, g)
        ok &= run_case(c, "kmeans%d" % universe, r, 8, km, iters)
        if universe == 16:
            # what the stock node pays first: the whole File to the host
            f = capi.DevFile(r.data_ptr(), r.shape[0], 40, 0)
            host = c.host_alloc(r.numel() * 4)
            blocks = (capi.Block * 1)()
            blocks[0].data, blocks[0].bytes = host.ctypes.data, host.nbytes
            med, best = timed(c, lambda: c.ck(c.L.tg_dev_file_fetch(c.h, C.byref(f), blocks, 1)), max(3, iters // 3))
            print("fetch      %.1e x 40 B to page-locked host memory: %.2f ms (min %.2f), %.1f GB/s"
                  % (r.shape[0], med, best, host.nbytes / best / 1e6), flush=True)
            c.host_free(host)
        del r
        torch.cuda.empty_cache()
    li = [(8, 1, capi.OP_SUM_U64), (16, 1, capi.OP_SUM_F64), (24, 1, capi.OP_SUM_F64), (32, 1, capi.OP_SUM_F64)]
    r, _ = records(60_000_000, 176, 1, 4, li, g)
    ok &= run_case(c, "tpch", r, 1, li, iters)
    del r
    torch.cuda.empty_cache()
    mk = [(8, 2, capi.OP_SUM_F64), (24, 1, capi.OP_SUM_U64)]
    r, _ = records(100_000_000, 32, 8, 1 << 26, mk, g)
    ok &= run_case(c, "manykeys", r, 8, mk, iters)
    del r
    torch.cuda.empty_cache()
    pr = [(8, 1, capi.OP_SUM_U64)]
    r, _ = records(100_000_000, 16, 8, 1 << 26, pr, g)
    ok &= run_case(c, "pairs", r, 8, pr, iters)
    out, m = C.c_void_p(), C.c_size_t()
    kd = capi.KVDesc(16, capi.OP_SUM_U64)
    med, best = timed(c, lambda: c.ck(c.L.tg_reduce_by_key(c.h, C.byref(kd), r.data_ptr(), r.shape[0], C.byref(out), C.byref(m))), iters)
    m_ref, want = model_checksum(c, r, pr)
    pok = m.value == m_ref and c.checksum(out.value, m.value, 16) == want       # (order-independent: the pair path's table order)
    print("pairs      the same 1e8 pairs through tg_reduce_by_key: %.2f ms (min %.2f), %d keys; %s"
          % (med, best, m.value, "equal to the model" if pok else "DIFFERENT from the model"), flush=True)
    ok &= pok
    c.close()
    print("ALL OK" if ok else "SOME CHECK FAILED", flush=True)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
