"""Worker of test_gpu_window.py::test_window_on_n_gpus: one process per GPU (torchrun), runs tg_window on shards placed as the
reference's workers held them (tests/golden/reference_outputs_window.npz at p = world, where that worker count was recorded;
otherwise its own sharding) and checks each rank's outputs against its slice of the model (double sums against the emulated
bracketing, bit for bit), and their counts.  A halo that spans several predecessors comes from shards smaller than k - 1.
Exit code 0 and MULTI_GPU_WINDOW_OK = parity."""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch.distributed as dist  # noqa: E402

import window_ref as W  # noqa: E402
from thrill_b200 import api, capi  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "reference_outputs_window.npz")


def want_rows(words, op, k, form):
    want = W.outputs(words, op, k, form)
    if op == W.OP_SUM_F64:
        want[:, 1] = W.emulate_sum(words[:, 1], k, form)
    return want


def run(tg, words, sizes, rank, op, pair, k, form):
    ib = 16 if pair else 8
    items = np.ascontiguousarray(words if pair else words[:, 1])
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(int)
    mine = items[off[rank]:off[rank + 1]]
    d = tg.to_device(mine) if len(mine) else None
    out, n = C.c_void_p(), C.c_size_t()
    tg.ck(tg.L.tg_window(tg.h, C.byref(capi.ScanDesc(ib, op)), d, len(mine), k, form, C.byref(out), C.byref(n)))
    raw = tg.download(out.value, n.value * ib).view(np.uint64) if n.value else np.zeros(0, np.uint64)
    if d is not None:
        tg.free(d)
    got = raw.reshape(-1, 2) if pair else np.stack([np.zeros(len(raw), np.uint64), raw], axis=1)
    cnt = W.counts(form, k, sizes)
    lo = sum(cnt[:rank])
    want = want_rows(words, op, k, form)[lo:lo + cnt[rank]]
    assert n.value == cnt[rank] and W.same(got, want, op), (op, pair, k, form, sizes, rank)


def main():
    ctx = api.Context.from_env(rng_seed=5)
    rank, world = ctx.my_rank(), ctx.num_workers()
    tg = ctx.tg
    checked = 0
    if world in W.WORKERS:
        for c in W.load_fixtures(GOLDEN)[::3]:
            run(tg, c["items"], c["shards"][world], rank, c["op"], c["pair"], c["k"], c["form"])
            checked += 1
    rng = np.random.RandomState(world)
    for k in (2, 33, 4096):
        n = 3 * k + 5000
        words = np.stack([rng.randint(0, 1 << 62, n).astype(np.uint64),
                          rng.standard_normal(n).view(np.uint64)], axis=1)
        small = max(1, (k - 1) // 3)
        sizes = [small] * (world - 1) + [n - small * (world - 1)]
        for op in (W.OP_SUM_F64, W.OP_MAX_F64, W.OP_SUM_U64):
            for form in (W.FULL, W.PARTIAL, W.DISJOINT):
                run(tg, words, sizes, rank, op, True, k, form)
                checked += 1
    tg.barrier()
    if rank == 0:
        print("MULTI_GPU_WINDOW_OK world=%d cases=%d" % (world, checked), flush=True)
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
