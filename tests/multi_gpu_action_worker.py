"""Worker of test_gpu_action.py::test_action_on_n_gpus: one process per GPU (torchrun), runs tg_all_reduce on shards placed as the
reference's workers held them and checks the result against the reference's result at p = world in
tests/golden/reference_outputs_action.npz (uneven and empty shards included; double sums against the exact sum within the rounding
bound), with the same value on every rank; then a shard of a real 2^30-item buffer on rank 0: TG_ERR_TOO_LARGE on every rank.
Exit code 0 and MULTI_GPU_ACTION_OK = parity."""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import action_ref as A  # noqa: E402
from test_gpu_action import check_sum_f64  # noqa: E402
from thrill_b200 import api, capi  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "reference_outputs_action.npz")
TG_ERR_TOO_LARGE = -4


def run(tg, case, shard):
    ib = 16 if case.pair else 8
    d = tg.to_device(shard)
    out = np.zeros(2, np.uint64)
    ini = None if case.initial is None else np.array(case.initial if case.pair else [case.initial[1]], np.uint64)
    st = tg.L.tg_all_reduce(tg.h, C.byref(capi.ScanDesc(ib, case.op)), d, len(shard), None if ini is None else ini.ctypes.data,
                            out.ctypes.data)
    assert st == 0, (case.name, st, tg.L.tg_last_error(tg.h))
    tg.free(d)
    return (int(out[0]), int(out[1])) if case.pair else (0, int(out[0]))


def main():
    ctx = api.Context.from_env(rng_seed=5)
    rank, world = ctx.my_rank(), ctx.num_workers()
    tg = ctx.tg
    g = A.Golden(GOLDEN)
    checked = 0
    for name in A.case_names(g):
        case = A.Case(g, name)
        if world not in case.ps:
            continue
        got = run(tg, case, case.shards(world)[rank])
        want = case.result(world)
        if case.op == A.OP_SUM_F64:
            check_sum_f64(got, case.shards(world), case.pair, case.initial)
        else:
            assert got == want, (name, rank, got, want)
        # the same value on every rank
        t = torch.tensor([got[0] & ((1 << 63) - 1), got[1] & ((1 << 63) - 1), got[0] >> 63, got[1] >> 63], dtype=torch.int64)
        lo, hi = t.clone(), t.clone()
        dist.all_reduce(lo, op=dist.ReduceOp.MIN)
        dist.all_reduce(hi, op=dist.ReduceOp.MAX)
        assert torch.equal(lo, hi), (name, rank)
        checked += 1
    assert checked >= 20

    # one worker holds a real buffer of 2^30 items: every rank returns TG_ERR_TOO_LARGE, and the ctx keeps working
    n = (1 << 30) if rank == 0 else 16
    big = torch.empty(n, dtype=torch.int64, device="cuda:%d" % tg.device)
    out = np.zeros(2, np.uint64)
    st = tg.L.tg_all_reduce(tg.h, C.byref(capi.ScanDesc(8, capi.OP_SUM_U64)), big.data_ptr(), n, None, out.ctypes.data)
    assert st == TG_ERR_TOO_LARGE, st
    del big
    torch.cuda.empty_cache()
    x = np.arange(1000 * (rank + 1), dtype=np.uint64)
    d = tg.to_device(x)
    tg.ck(tg.L.tg_all_reduce(tg.h, C.byref(capi.ScanDesc(8, capi.OP_SUM_U64)), d, len(x), None, out.ctypes.data))
    assert int(out[0]) == sum(sum(range(1000 * (r + 1))) for r in range(world))
    tg.free(d)

    tg.barrier()
    if rank == 0:
        print("MULTI_GPU_ACTION_OK world=%d cases=%d" % (world, checked), flush=True)
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
