"""Sample and BernoulliSample on one H100: tg_sample / tg_bernoulli_sample, their _file and _select forms and the Python mirror,
bit for bit against the numpy model of sample_ref.py.  Items carry their global position, so an output names the positions it
kept.  Item sizes 4 to 256 bytes, sizes around the 4096-position tile, every kind of s and p, 1 to 16 simulated workers with
empty shards (the concatenation is the same for every sharding), host and device Files (left intact), argument errors and the
size limit (refused before any read), a 1e8-item case, one uniformity check, the multi-GPU worker and the in-Thrill test binary
where the machine has what they need.  pytest -m gpu."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
from scipy import stats

import sample_ref as S
from gpu_util import make_blocks

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
TG_ERR_ARG, TG_ERR_TOO_LARGE = -3, -4
TILE = 4096
ITEM_BYTES = [4, 8, 16, 24, 100, 256]
SEEDS = [0, (1 << 64) - 1, 0x1234567890ABCDEF]
PS = [0.0, 2.0 ** -53, 1e-6, 0.05, 0.5, 1 - 2.0 ** -53, 1.0]


def _capi():
    from thrill_b200 import capi
    return capi


@pytest.fixture(scope="module")
def ctx():
    c = _capi().Ctx(0)
    yield c
    c.close()


def make_items(N, ib, base=0):
    """(N, ib // 4) uint32 words: word 0 the low 32 bits of the global position, word 1 (if any) the high ones, the rest a hash"""
    w = ib // 4
    g = np.arange(base, base + N, dtype=np.uint64)
    out = np.empty((N, w), np.uint32)
    out[:, 0] = (g & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    if w > 1:
        out[:, 1] = (g >> np.uint64(32)).astype(np.uint32)
    if w > 2:
        h = S.mix(g[:, None] * np.uint64(w) + np.arange(w - 2, dtype=np.uint64)[None, :] + np.uint64(1))
        out[:, 2:] = (h & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    return out


def _download(ctx, dptr, n, ib):
    if not n:
        return np.zeros((0, ib // 4), np.uint32)
    return ctx.download(dptr, n * ib).view(np.uint32).reshape(n, ib // 4)


def run_one(ctx, d, items, bern, param, seed):
    """tg_sample / tg_bernoulli_sample on one worker over the device copy d of items"""
    N, ib = items.shape[0], items.shape[1] * 4
    out, n = C.c_void_p(), C.c_size_t()
    fn = ctx.L.tg_bernoulli_sample if bern else ctx.L.tg_sample
    ctx.ck(fn(ctx.h, ib, d, N, param, seed, C.byref(out), C.byref(n)))
    return _download(ctx, out.value, n.value, ib)


def model_mask(bern, N, param, seed):
    return S.bernoulli_mask(seed, N, param) if bern else S.sample_mask(seed, N, param)


def s_values(N):
    return sorted({0, 1, 10, max(N - 1, 0), N, N + 1, 1 << 40})


@pytest.mark.parametrize("ib", ITEM_BYTES)
def test_sample_one_worker(ctx, ib):
    for N in (0, 1, 2, TILE - 1, TILE, TILE + 1, 1_000_000) + ((10_000_000,) if ib in (8, 16) else ()):
        items = make_items(N, ib)
        d = ctx.to_device(items) if N else None
        for seed in SEEDS:
            for s in s_values(N):
                got = run_one(ctx, d, items, False, s, seed)
                want = items[S.sample_mask(seed, N, s)]
                assert got.shape == want.shape and np.array_equal(got, want), (ib, N, s, seed)
        if d is not None:
            assert np.array_equal(ctx.download(d, items.nbytes).view(np.uint32).reshape(items.shape), items)
            ctx.free(d)


@pytest.mark.parametrize("ib", ITEM_BYTES)
def test_bernoulli_one_worker(ctx, ib):
    for N in (0, 1, 2, TILE - 1, TILE, TILE + 1, 1_000_000) + ((10_000_000,) if ib in (8, 16) else ()):
        items = make_items(N, ib)
        d = ctx.to_device(items) if N else None
        for seed in SEEDS:
            for p in PS:
                got = run_one(ctx, d, items, True, p, seed)
                want = items[S.bernoulli_mask(seed, N, p)]
                assert got.shape == want.shape and np.array_equal(got, want), (ib, N, p, seed)
        if d is not None:
            assert np.array_equal(ctx.download(d, items.nbytes).view(np.uint32).reshape(items.shape), items)
            ctx.free(d)


def run_select(ctx, items, sizes, bern, params, seeds):
    """workers 0..p-1 through the _select form: the per-worker outputs"""
    ib = items.shape[1] * 4
    p = len(sizes)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(int)
    devs = [ctx.to_device(items[off[r]:off[r + 1]]) if sizes[r] else None for r in range(p)]
    ptrs = (C.c_void_p * p)(*devs)
    ns = (C.c_size_t * p)(*sizes)
    pr = (C.c_double * p)(*params) if bern else (C.c_uint64 * p)(*params)
    sd = (C.c_uint64 * p)(*seeds)
    fn = ctx.L.tg_bernoulli_sample_select if bern else ctx.L.tg_sample_select
    parts = []
    for r in range(p):
        out, n = C.c_void_p(), C.c_size_t()
        ctx.ck(fn(ctx.h, ib, ptrs, ns, p, r, pr, sd, C.byref(out), C.byref(n)))
        parts.append(_download(ctx, out.value, n.value, ib))
    for r, d in enumerate(devs):
        if d is not None:
            assert np.array_equal(ctx.download(d, sizes[r] * ib).view(np.uint32).reshape(sizes[r], -1), items[off[r]:off[r + 1]])
            ctx.free(d)
    return parts


def shardings(N, p, rng):
    """an even sharding, one with empty workers, and all items on one worker"""
    even = [N * (r + 1) // p - N * r // p for r in range(p)]
    cuts = np.sort(rng.randint(0, N + 1, p - 1))
    rand = np.diff(np.concatenate([[0], cuts, [N]])).astype(int).tolist()
    if p > 2:
        rand[1] += rand[2]
        rand[2] = 0
    one = [0] * p
    one[p // 2] = N
    return [even, rand, one]


@pytest.mark.parametrize("p", [1, 2, 3, 5, 8, 16])
def test_select_every_sharding(ctx, p):
    rng = np.random.RandomState(p)
    for ib in (8, 24):
        for N in (0, 7, TILE + 1, 300_000):
            items = make_items(N, ib)
            for sizes in shardings(N, p, rng):
                for seed in (0, (1 << 64) - 1):
                    for s in (0, 1, 10, max(N - 1, 0), N, 1 << 40):
                        mask = S.sample_mask(seed, N, s)
                        got = run_select(ctx, items, sizes, False, [s] * p, [seed] + [(seed + 1 + r) % (1 << 64) for r in range(p - 1)])
                        want = S.split(items, mask, sizes)
                        assert all(np.array_equal(g, w) for g, w in zip(got, want)), (ib, N, sizes, s, seed)
                    for q in (0.0, 1e-6, 0.3, 1.0):
                        got = run_select(ctx, items, sizes, True, [q] * p, [seed] * p)
                        want = S.split(items, S.bernoulli_mask(seed, N, q), sizes)
                        assert all(np.array_equal(g, w) for g, w in zip(got, want)), (ib, N, sizes, q, seed)


@pytest.mark.parametrize("bern", [False, True])
def test_file_forms(ctx, bern):
    """a host File in odd-sized Blocks (items straddle them) and a device File (left intact), results fetched and detached"""
    capi = _capi()
    for ib in (4, 16, 100):
        N = 50_000
        items = make_items(N, ib)
        param, seed = (0.25 if bern else 777), 99
        want = items[model_mask(bern, N, param, seed)]
        fn = ctx.L.tg_bernoulli_sample_file if bern else ctx.L.tg_sample_file
        blocks, nb, raw = make_blocks(capi, items, 1000 + 4 * 7 + 1)
        n_out = C.c_size_t()
        ctx.ck(fn(ctx.h, ib, C.byref(capi.MergeInput(None, C.cast(blocks, C.POINTER(capi.Block)), nb)), param, seed, C.byref(n_out)))
        out = np.empty(n_out.value * ib, np.uint8)
        ob, onb, _ = make_blocks(capi, out, 4096 + 3)
        ctx.ck(ctx.L.tg_fetch_output(ctx.h, C.cast(ob, C.POINTER(capi.Block)), onb))
        assert np.array_equal(out.view(np.uint32).reshape(-1, ib // 4), want)
        d = ctx.to_device(items)
        dev = capi.DevFile(d, N, ib, 0)
        ctx.ck(fn(ctx.h, ib, C.byref(capi.MergeInput(C.pointer(dev), None, 0)), param, seed, C.byref(n_out)))
        res = capi.DevFile()
        ctx.ck(ctx.L.tg_output_detach(ctx.h, C.byref(res)))
        assert res.items == len(want) and res.item_bytes == ib
        assert np.array_equal(_download(ctx, res.dptr, res.items, ib), want)
        ctx.ck(ctx.L.tg_dev_file_free(ctx.h, C.byref(res)))
        assert np.array_equal(ctx.download(d, items.nbytes).view(np.uint32).reshape(items.shape), items)
        # a device File of another item size is refused
        bad = capi.DevFile(d, N, ib + 4, 0)
        assert fn(ctx.h, ib, C.byref(capi.MergeInput(C.pointer(bad), None, 0)), param, seed, C.byref(n_out)) == TG_ERR_ARG
        ctx.free(d)


def test_python_mirror(ctx):
    from thrill_b200 import api
    c = api.Context(rank=0, nranks=1, device=0, rng_seed=5)
    try:
        x = np.arange(100_000, dtype=np.uint64)
        got = api.DIA(c, x).Sample(1000, seed=3).items
        assert np.array_equal(got, x[S.sample_mask(3, len(x), 1000)])
        got = api.DIA(c, x).BernoulliSample(0.1, seed=4).items
        assert np.array_equal(got, x[S.bernoulli_mask(4, len(x), 0.1)])
        rec = make_items(5000, 100).view(np.uint8).reshape(5000, 100)
        got = api.DIA(c, rec).Sample(17, seed=8).items
        assert np.array_equal(got, rec[S.sample_mask(8, 5000, 17)])
        # without a seed: the context's next seed, so two draws in a row differ
        a = api.DIA(c, x).Sample(1000).items
        b = api.DIA(c, x).Sample(1000).items
        assert len(a) == len(b) == 1000 and not np.array_equal(a, b)
        with pytest.raises(_capi().ThrillGpuError):
            api.DIA(c, x).BernoulliSample(1.5)
    finally:
        c.close()


def test_fixture_deterministic_cases(ctx):
    """the stock operators' deterministic cases (tests/golden/reference_outputs_sample.npz) through the _select form: s >= N and
    N = 0 at 1 to 4 workers, BernoulliSample(1) and (0); Sample(s < n) on one worker keeps s of its items"""
    import test_sample_ref as R
    n = 0
    for sizes, mode, param, exact, stock in R.det_cases(R.load_fixture()):
        items = np.arange(sum(sizes), dtype=np.uint64).reshape(-1, 1).view(np.uint32).reshape(-1, 2)
        for seed in (0, (1 << 64) - 1):
            got = run_select(ctx, items, sizes, bool(mode), [param] * len(sizes), [seed] * len(sizes))
            got = [g.reshape(-1).view(np.uint64).astype(np.int64) for g in got]
            if exact:
                assert all(np.array_equal(g, s) for g, s in zip(got, stock)), (sizes, mode, param)
            else:
                assert len(got[0]) == len(stock[0]) == param and len(np.unique(got[0])) == param
        n += 1
    assert n == 21


# ---- errors and the size limit -------------------------------------------------------------------------------------------------
def test_argument_errors(ctx):
    d = ctx.to_device(np.arange(1024, dtype=np.uint64))
    out, n = C.c_void_p(), C.c_size_t()
    for ib in (0, 2, 3, 6, 260, 512):
        assert ctx.L.tg_sample(ctx.h, ib, d, 16, 4, 1, C.byref(out), C.byref(n)) == TG_ERR_ARG
        assert ctx.L.tg_bernoulli_sample(ctx.h, ib, d, 16, 0.5, 1, C.byref(out), C.byref(n)) == TG_ERR_ARG
    for q in (float("nan"), -0.1, -0.0 - 1e-300, 1.5, float("inf"), -float("inf")):
        assert ctx.L.tg_bernoulli_sample(ctx.h, 8, d, 16, q, 1, C.byref(out), C.byref(n)) == TG_ERR_ARG
    assert ctx.L.tg_sample(ctx.h, 8, None, 16, 4, 1, C.byref(out), C.byref(n)) == TG_ERR_ARG
    # the ranks disagree on s or p: every rank is refused; seeds may differ (rank 0's wins)
    ptrs = (C.c_void_p * 3)(d, d, d)
    ns = (C.c_size_t * 3)(100, 0, 50)
    sd = (C.c_uint64 * 3)(1, 2, 3)
    for r in range(3):
        assert ctx.L.tg_sample_select(ctx.h, 8, ptrs, ns, 3, r, (C.c_uint64 * 3)(5, 5, 6), sd, C.byref(out), C.byref(n)) == TG_ERR_ARG
        assert ctx.L.tg_bernoulli_sample_select(ctx.h, 8, ptrs, ns, 3, r, (C.c_double * 3)(0.5, 0.25, 0.5), sd, C.byref(out),
                                                C.byref(n)) == TG_ERR_ARG
        nan = (C.c_double * 3)(float("nan"), float("nan"), float("nan"))
        assert ctx.L.tg_bernoulli_sample_select(ctx.h, 8, ptrs, ns, 3, r, nan, sd, C.byref(out), C.byref(n)) == TG_ERR_ARG
    # no workers, rank >= p, more than 16 workers
    for p, r in ((0, 0), (3, 3), (17, 0)):
        assert ctx.L.tg_sample_select(ctx.h, 8, ptrs, ns, p, r, (C.c_uint64 * 3)(5, 5, 5), sd, C.byref(out), C.byref(n)) == TG_ERR_ARG
    ctx.free(d)


def test_size_limit(ctx):
    """2^30 items on a worker is refused on every rank before any read (the pointers cover 8 KB only)"""
    d = ctx.to_device(np.arange(1024, dtype=np.uint64))
    out, n = C.c_void_p(), C.c_size_t()
    for ib in (4, 8, 256):
        assert ctx.L.tg_sample(ctx.h, ib, d, 1 << 30, 10, 1, C.byref(out), C.byref(n)) == TG_ERR_TOO_LARGE
        assert ctx.L.tg_bernoulli_sample(ctx.h, ib, d, 1 << 30, 0.5, 1, C.byref(out), C.byref(n)) == TG_ERR_TOO_LARGE
        ptrs = (C.c_void_p * 3)(d, d, d)
        ns = (C.c_size_t * 3)(1, 1 << 30, 1)
        sd = (C.c_uint64 * 3)(1, 1, 1)
        for r in range(3):
            # (the limit is decided before the disagreement on s)
            assert ctx.L.tg_sample_select(ctx.h, ib, ptrs, ns, 3, r, (C.c_uint64 * 3)(10, 11, 10), sd, C.byref(out),
                                          C.byref(n)) == TG_ERR_TOO_LARGE
            assert ctx.L.tg_bernoulli_sample_select(ctx.h, ib, ptrs, ns, 3, r, (C.c_double * 3)(0.5, 0.5, 0.5), sd, C.byref(out),
                                                    C.byref(n)) == TG_ERR_TOO_LARGE
    ctx.free(d)
    items = make_items(1000, 8)
    d = ctx.to_device(items)
    assert np.array_equal(run_one(ctx, d, items, False, 10, 2), items[S.sample_mask(2, 1000, 10)])
    ctx.free(d)


# ---- scale and uniformity ------------------------------------------------------------------------------------------------------
def test_1e8_u64(ctx):
    N = 100_000_000
    x = np.arange(N, dtype=np.uint64)
    d = ctx.to_device(x)
    out, n = C.c_void_p(), C.c_size_t()
    k = S.keys(11, x)
    for s in (10, 50_000_000):
        ctx.ck(ctx.L.tg_sample(ctx.h, 8, d, N, s, 11, C.byref(out), C.byref(n)))
        got = ctx.download(out.value, n.value * 8).view(np.uint64)
        K = np.partition(k, s - 1)[s - 1]
        assert n.value == s and np.array_equal(got, x[k <= K]), s
    ctx.ck(ctx.L.tg_bernoulli_sample(ctx.h, 8, d, N, 0.5, 11, C.byref(out), C.byref(n)))
    got = ctx.download(out.value, n.value * 8).view(np.uint64)
    assert np.array_equal(got, x[(k >> np.uint64(11)) < np.uint64(1 << 52)])
    ctx.free(d)


def test_uniform_positions(ctx):
    """Sample(1e5) of 1e7: the kept positions over 1000 buckets of 10^4 positions are consistent with uniform"""
    N, s = 10_000_000, 100_000
    x = np.arange(N, dtype=np.uint64)
    d = ctx.to_device(x)
    out, n = C.c_void_p(), C.c_size_t()
    ctx.ck(ctx.L.tg_sample(ctx.h, 8, d, N, s, 2024, C.byref(out), C.byref(n)))
    got = ctx.download(out.value, n.value * 8).view(np.uint64)
    ctx.free(d)
    assert len(got) == s and len(np.unique(got)) == s
    _, pv = stats.chisquare(np.bincount((got // np.uint64(N // 1000)).astype(np.int64), minlength=1000))
    assert pv > 1e-4, pv


# ---- several GPUs --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 4, 8])
def test_sample_on_n_gpus(world):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(29971 + world), os.path.join(HERE, "multi_gpu_sample_worker.py")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert res.returncode == 0 and "MULTI_GPU_SAMPLE_OK" in res.stdout, res.stdout[-3000:] + res.stderr[-3000:]


# ---- inside a real Thrill job (GpuSampleNode) ----------------------------------------------------------------------------------
HOST_BIN = os.path.join(ROOT, "oracle", "_ref", "host", "gpu_sample_test")


def _host_run(workers):
    env = dict(os.environ, THRILL_NET="mock", THRILL_LOCAL="1", THRILL_WORKERS_PER_HOST=str(workers), THRILL_LOG="")
    res = subprocess.run([HOST_BIN], env=env, capture_output=True, text=True, timeout=900)
    lines = [l for l in res.stdout.splitlines() if l.startswith(("PASS", "FAIL"))]
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert len(lines) == 5 and all(l.startswith("PASS") for l in lines), lines


@pytest.mark.skipif(not os.path.exists(HOST_BIN), reason="oracle/_ref/host/gpu_sample_test not built (make -C tests/host -f gpu_sample_test.mk)")
def test_sample_inside_thrill_single_worker():
    _host_run(1)


@pytest.mark.skipif(not os.path.exists(HOST_BIN), reason="oracle/_ref/host/gpu_sample_test not built")
def test_sample_inside_thrill_two_workers_two_gpus():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _host_run(2)
