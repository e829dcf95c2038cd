"""Worker of test_gpu_scan.py::test_scan_on_n_gpus: one process per GPU (torchrun), runs tg_prefix_sum / tg_zip_with_index on
shards placed as the reference's workers held them and checks this worker's rows against the reference's worker `rank` at
p = world in tests/golden/reference_outputs_scan.npz (uneven and empty shards included; double sums within the tolerance of
test_gpu_scan.py), then a shard of a real 2^30-item buffer on rank 0: TG_ERR_TOO_LARGE on every rank.  Exit code 0 and
MULTI_GPU_SCAN_OK = parity."""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import scan_ref as S  # noqa: E402
from test_gpu_scan import assert_f64_close  # noqa: E402
from thrill_b200 import api, capi  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "reference_outputs_scan.npz")
TG_ERR_TOO_LARGE = -4


def run(tg, case, shard):
    d = tg.to_device(shard)
    out, n = C.c_void_p(), C.c_size_t()
    if case.op is None:
        st = tg.L.tg_zip_with_index(tg.h, d, len(shard), int(case.mode == "zip_first"), C.byref(out), C.byref(n))
        ib = 16
    else:
        ib = 16 if case.pair else 8
        ini = np.array(case.initial if case.pair else [case.initial[1]], np.uint64)
        st = tg.L.tg_prefix_sum(tg.h, C.byref(capi.ScanDesc(ib, case.op)), d, len(shard), ini.ctypes.data, int(case.inclusive),
                                C.byref(out), C.byref(n))
    assert st == 0, (case.name, st, tg.L.tg_last_error(tg.h))
    assert n.value == len(shard)
    res = tg.download(out.value, n.value * ib) if n.value else np.zeros(0, np.uint8)
    tg.free(d)
    return res.view(S.KV) if ib == 16 else res.view(np.uint64)


def main():
    ctx = api.Context.from_env(rng_seed=5)
    rank, world = ctx.my_rank(), ctx.num_workers()
    tg = ctx.tg
    g = np.load(GOLDEN)
    checked = 0
    for name in S.case_names(g):
        case = S.Case(g, name)
        if world not in case.ps:
            continue
        shard = case.shards(world)[rank]
        res = run(tg, case, shard)
        counts = case.counts(world)
        lo = sum(counts[:rank])
        ref = case.rows(world)[lo:lo + counts[rank]]
        rows = S.as_rows([res])
        rows[:, 0] = rank
        if case.op == S.OP_SUM_F64:
            assert np.array_equal(rows[:, :2], ref[:, :2]), name
            init = float(np.array([case.initial[1]], np.uint64).view(np.float64)[0])
            scale = S.f64_abs_prefix(case.shards(world), case.pair, init)[rank]
            assert_f64_close(rows[:, 2], ref[:, 2], scale)
        else:
            assert S.rows_equal(rows, ref), (name, rank)
        checked += 1
    assert checked >= 20

    # one worker holds a real buffer of 2^30 items: every rank returns TG_ERR_TOO_LARGE, and the ctx keeps working
    big = torch.empty((1 << 30) if rank == 0 else 16, dtype=torch.int64, device="cuda:%d" % tg.device)
    n = (1 << 30) if rank == 0 else 16
    out, m = C.c_void_p(), C.c_size_t()
    st = tg.L.tg_prefix_sum(tg.h, C.byref(capi.ScanDesc(8, capi.OP_SUM_U64)), big.data_ptr(), n, None, 1, C.byref(out), C.byref(m))
    assert st == TG_ERR_TOO_LARGE, st
    st = tg.L.tg_zip_with_index(tg.h, big.data_ptr(), n, 1, C.byref(out), C.byref(m))
    assert st == TG_ERR_TOO_LARGE, st
    del big
    torch.cuda.empty_cache()
    x = np.arange(1000 * (rank + 1), dtype=np.uint64)
    d = tg.to_device(x)
    tg.ck(tg.L.tg_prefix_sum(tg.h, C.byref(capi.ScanDesc(8, capi.OP_SUM_U64)), d, len(x), None, 0, C.byref(out), C.byref(m)))
    res = tg.download(out.value, m.value * 8).view(np.uint64)
    shards = [np.arange(1000 * (r + 1), dtype=np.uint64) for r in range(world)]
    assert np.array_equal(res, S.prefix_sum(shards, "sum_u64", inclusive=False)[rank])
    tg.free(d)

    tg.barrier()
    if rank == 0:
        print("MULTI_GPU_SCAN_OK world=%d cases=%d" % (world, checked), flush=True)
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
