"""Host-side mirror of the reference's DIA<T> operator interface for the Sort / ReduceByKey path.

Mirrors (same names, argument meaning and error behaviour) the slice of thrill/api that drives the hot path:
    api::Run / Context                     thrill/api/context.hpp:243-377  (my_rank, num_workers)
    api::Generate(ctx, n, fn)              thrill/api/generate.hpp         (even range split over workers)
    DIA<T>::Sort(cmp) / SortStable(cmp)    thrill/api/sort.hpp:800-937
    DIA<T>::ReducePair(reduce_fn)          thrill/api/reduce_by_key.hpp:410-449
    DIA<T>::ReduceByKey(key_ex, reduce_fn) thrill/api/reduce_by_key.hpp:312-363 (pairs on .first; records on a KeyField with a
                                           FieldReduce)
    DIA<T>::Merge(second, cmp) / api::Merge thrill/api/merge.hpp:674-721
    DIA<T>::GroupByKey / GroupToIndex      thrill/api/group_by_key.hpp:419-428, group_to_index.hpp:257-290
    DIA<T>::PrefixSum / ExPrefixSum        thrill/api/dia.hpp:1850, :1867 (api/prefix_sum.hpp, ex_prefix_sum.hpp)
    DIA<T>::ZipWithIndex(zip_function)     thrill/api/zip_with_index.hpp:140-152
    api::InnerJoin(l, r, key1, key2, fn)   thrill/api/inner_join.hpp:700-827 (pairs on .first; records on a KeyField)
    DIA<T>::Sum / Min / Max / AllReduce    thrill/api/sum.hpp, min.hpp, max.hpp, all_reduce.hpp
    DIA<T>::HyperLogLog<p>                 thrill/api/hyperloglog.hpp:62-72 (the registers, not the estimate)
    DIA<T>::Window(k, f[, partial_f])      thrill/api/window.hpp:284-380, :524-564 (the left fold of each window)
    DIA<T>::Sample / BernoulliSample       thrill/api/sample.hpp:37-140, bernoulli_sample.hpp:27-77 (by global position)
    DIA<T>::Size / AllGather / Gather      thrill/api/size.hpp, all_gather.hpp, gather.hpp
A DIA here holds its local shard as a host numpy array — the stand-in for a data::File whose Blocks are
1 MiB ByteBlocks (data/byte_block.cpp:23-24, data/block_writer.hpp:405-420).  Operators hand the Blocks to the
C ABI (tg_sort_file / tg_reduce_file / tg_fetch_output): exactly what thrill_b200/host/gpu_sort_node.hpp does
from C++.  Like the C++ host shim, only a closed set of functors is recognised (SURVEY.md §7 "UDFs");
anything else raises — there is no CPU fallback.

torch.distributed is used only as the control plane between the one-process-per-GPU workers (what Thrill's
net::FlowControlChannel does): broadcasting the NCCL id and gathering results for AllGather().
"""
import ctypes as C
import os

import numpy as np

from . import capi

KV = np.dtype([("key", "<u8"), ("val", "<u8")])          # std::pair<uint64_t, 8-byte value>, member-wise
BLOCK_BYTES = 1 << 20                                      # largest ByteBlock BlockWriter produces by default


class _Functor(object):
    def __init__(self, name, code=None):
        self.name, self.code = name, code

    def __repr__(self):
        return "<thrill_b200 functor %s>" % self.name


# recognised comparators (std::less<T> / std::greater<T>) and reduce functions
Less = _Functor("std::less")
Greater = _Functor("std::greater")
PlusDouble = _Functor("std::plus<double>", capi.OP_SUM_F64)
PlusU64 = _Functor("std::plus<uint64_t>", capi.OP_SUM_U64)
MinU64 = _Functor("min<uint64_t>", capi.OP_MIN_U64)
MaxU64 = _Functor("max<uint64_t>", capi.OP_MAX_U64)
MinDouble = _Functor("min<double>", capi.OP_MIN_F64)
MaxDouble = _Functor("max<double>", capi.OP_MAX_F64)
First = _Functor("first", capi.OP_FIRST)
KeyIsFirst = _Functor("pair.first")                       # the key extractor ReducePair builds (:444-449)
# recognised join functions of InnerJoin on pair DIAs
JoinKeyValues = _Functor("(l, r) -> tuple(l.first, l.second, r.second)", capi.JOIN_KEY_VALUES)
JoinValues = _Functor("(l, r) -> pair(l.second, r.second)", capi.JOIN_VALUES)
KEY_V1_V2 = np.dtype([("key", "<u8"), ("v1", "<u8"), ("v2", "<u8")])     # std::tuple<uint64_t, V1, V2>, member-wise
V1_V2 = np.dtype([("v1", "<u8"), ("v2", "<u8")])                         # std::pair<V1, V2>
# the join function of InnerJoin on records: (l, r) -> std::pair<L, R>, the left item's bytes then the right item's
JoinPair = _Functor("(l, r) -> pair(l, r)")


def KeyField(offset, nbytes):
    """thrill_gpu::KeyField: the key extractor of InnerJoin on records, the unsigned little-endian integer of nbytes (1..8) bytes at
    byte offset `offset` of an item, zero-extended to uint64_t"""
    f = _Functor("KeyField<%d, %d>" % (offset, nbytes))
    f.key_offset, f.key_bytes = int(offset), int(nbytes)
    return f


def FieldReduce(runs):
    """thrill_gpu::FieldReduce: the reduce function of ReduceByKey on records, given as at most 8 field runs (offset, count, f):
    `count` consecutive 8-byte fields from byte `offset` (a multiple of 4), each folded by f, one of PlusDouble, PlusU64, MinU64,
    MaxU64, MinDouble, MaxDouble.  Every other byte of a result comes from the group's first item.  No runs keeps one item per key."""
    runs = [tuple(r) for r in runs]
    for r in runs:
        if len(r) != 3 or not isinstance(r[2], _Functor) or r[2].code is None or r[2] is First:
            raise capi.ThrillGpuError("FieldReduce: run %r is not (offset, count, reduce function)" % (r,))
    f = _Functor("FieldReduce<%s>" % ", ".join("{%d, %d, %s}" % (o, c, fn.name) for o, c, fn in runs))
    f.runs = [(int(o), int(c), fn.code) for o, c, fn in runs]
    return f


def ScanSecond(value_function):
    """thrill_gpu::ScanSecond<F>: the sum function of PrefixSum and AllReduce on pair<uint64_t, 8-byte value>, a + b = (b.first,
    F(a.second, b.second)), with F one of PlusU64, MinU64, MaxU64, PlusDouble (and for AllReduce MinDouble, MaxDouble)"""
    if value_function not in (PlusU64, MinU64, MaxU64, PlusDouble, MinDouble, MaxDouble):
        raise capi.ThrillGpuError("ScanSecond: %r is not a sum function the GPU path recognises" % (value_function,))
    f = _Functor("ScanSecond<%s>" % value_function.name, value_function.code)
    f.on_second = True
    return f


# recognised zip functions of ZipWithIndex on 8-byte items: (index, item) or (item, index), as KV items
IndexFirst = _Functor("(item, index) -> pair(index, item)")
IndexSecond = _Functor("(item, index) -> pair(item, index)")


def bind_to_gpu_numa_node(device):
    """Run this worker process on the CPUs next to its GPU (nvidia-smi topo -m "CPU Affinity"): the pinned staging
    buffers it allocates afterwards, and the copies it issues, stay on the GPU's NUMA node.  What a Thrill launcher does
    with numactl per worker; without it eight workers share one node's memory controllers for their PCIe traffic."""
    try:
        import pynvml
        pynvml.nvmlInit()
        # NVML counts physical GPUs; CUDA ordinals go through CUDA_VISIBLE_DEVICES
        vis = [v.strip() for v in os.environ.get("CUDA_VISIBLE_DEVICES", "").split(",") if v.strip()]
        if vis and device < len(vis):
            h = pynvml.nvmlDeviceGetHandleByUUID(vis[device]) if vis[device].startswith("GPU-") else \
                pynvml.nvmlDeviceGetHandleByIndex(int(vis[device]))
        else:
            h = pynvml.nvmlDeviceGetHandleByIndex(device)
        ncpu = os.cpu_count() or 1
        mask = pynvml.nvmlDeviceGetCpuAffinity(h, (ncpu + 63) // 64)
        cpus = {i for i in range(ncpu) if (mask[i // 64] >> (i % 64)) & 1} & os.sched_getaffinity(0)
        if cpus:
            os.sched_setaffinity(0, cpus)
            return sorted(cpus)
    except Exception:          # noqa: BLE001  (no NVML, no permission: run unbound)
        pass
    return None


class Context(object):
    """One worker = one GPU (api/context.hpp:243-245)."""

    def __init__(self, rank=0, nranks=1, device=None, unique_id=None, rng_seed=None):
        self._rank, self._n = rank, nranks
        self.tg = capi.Ctx(device=rank if device is None else device, rank=rank, nranks=nranks, unique_id=unique_id)
        # the reference seeds each worker's rng from std::random_device (api/context.cpp:1190)
        self.rng_seed = int.from_bytes(os.urandom(8), "little") if rng_seed is None else rng_seed
        self._op_counter = 0

    @classmethod
    def from_env(cls, rng_seed=None):
        """one process per GPU under torchrun: RANK / LOCAL_RANK / WORLD_SIZE, id broadcast over torch.distributed"""
        rank = int(os.environ.get("RANK", "0"))
        world = int(os.environ.get("WORLD_SIZE", "1"))
        local = int(os.environ.get("LOCAL_RANK", str(rank)))
        uid = None
        if world > 1 and os.environ.get("TG_NUMA_BIND", "1") != "0":
            bind_to_gpu_numa_node(local)
        if world > 1:
            import torch.distributed as dist
            if not dist.is_initialized():
                dist.init_process_group("gloo")
            buf = [None]
            if rank == 0:
                raw = C.create_string_buffer(128)
                capi.check(capi.lib().tg_get_unique_id(raw))
                buf[0] = raw.raw
            dist.broadcast_object_list(buf, src=0)
            uid = buf[0]
        return cls(rank, world, device=local, unique_id=uid, rng_seed=rng_seed)

    def my_rank(self):
        return self._rank

    def num_workers(self):
        return self._n

    def close(self):
        self.tg.close()

    def _next_seed(self):
        self._op_counter += 1
        return (self.rng_seed + 0x9E3779B97F4A7C15 * self._op_counter) % (1 << 64)


def _local_range(n, p, r):
    """common::CalculateLocalRange (thrill/common/math.hpp): [r*n/p, (r+1)*n/p) in double arithmetic"""
    per = float(n) / float(p)
    lo = int(np.ceil(r * per))
    hi = min(n, int(np.ceil((r + 1) * per)))
    return lo, hi


def Generate(ctx, size, generator_function, dtype=np.uint64):
    """api::Generate: item i = generator_function(i) for the worker's index range; the generator here is
    vectorised: it receives a numpy array of global indices and returns the items."""
    lo, hi = _local_range(size, ctx.num_workers(), ctx.my_rank())
    idx = np.arange(lo, hi, dtype=np.uint64)
    items = np.ascontiguousarray(generator_function(idx))
    return DIA(ctx, items if dtype is None else items.astype(dtype, copy=False))


def _item_bytes(items):
    return items.dtype.itemsize if items.ndim == 1 else items.shape[1] * items.dtype.itemsize


def Merge(compare_function, *dias, **kw):
    """api::Merge(comparator, dia0, dia1, ...) (api/merge.hpp:674-713): 2..16 DIAs, each sorted by compare_function, of one
    item type the GPU path recognises (u64 or pair<u64, 8-byte value> ordered by the key; records are not supported)"""
    if len(dias) < 2:
        raise capi.ThrillGpuError("Merge: needs at least two DIAs")
    first = dias[0]
    for d in dias[1:]:
        if d.ctx is not first.ctx:
            raise capi.ThrillGpuError("Merge: the DIAs belong to different contexts")
        if d.items.dtype != first.items.dtype or d.items.shape[1:] != first.items.shape[1:]:
            raise capi.ThrillGpuError("Merge: the DIAs hold different item types (%r, %r)" % (first.items.dtype, d.items.dtype))
    desc, dtype = first._key_desc(compare_function)
    if desc.item_bytes not in (8, 16):
        raise capi.ThrillGpuError("Merge: %d-byte records are not supported by the GPU path" % desc.item_bytes)
    inputs = (capi.MergeInput * len(dias))()
    keep = []
    for j, d in enumerate(dias):
        blocks, nb = d._blocks(d.items)
        keep.append(blocks)
        inputs[j].blocks = C.cast(blocks, C.POINTER(capi.Block))
        inputs[j].nblocks = nb
    n_out = C.c_size_t()
    tg = first.ctx.tg
    tg.ck(tg.L.tg_merge_file(tg.h, C.byref(desc), inputs, len(dias), C.byref(n_out)))
    return DIA(first.ctx, first._fetch(n_out.value, dtype, desc.item_bytes, kw.get("_pinned_out")))


def InnerJoin(first, second, key_extractor1, key_extractor2, join_function, **kw):
    """api::InnerJoin(left, right, key_extractor1, key_extractor2, join_function) (api/inner_join.hpp:700-827), in two forms:
    on two DIAs of pair<uint64_t, 8-byte value> joined on .first (KeyIsFirst), JoinKeyValues gives KEY_V1_V2 items, JoinValues
    V1_V2 items; on two DIAs of fixed-size records (np.void or structured items, 4..1024 bytes in multiples of 4) joined on a
    KeyField(offset, nbytes) of each side (KeyIsFirst for pair items), JoinPair gives np.void items of left_bytes + right_bytes,
    the left item's bytes then the right item's.  Worker Hash128to64(0, key) % p holds a key's results, ordered by (key, left
    global position, right global position)."""
    if join_function is JoinPair:
        return _inner_join_records(first, second, key_extractor1, key_extractor2, kw.get("_pinned_out"))
    if key_extractor1 is not KeyIsFirst or key_extractor2 is not KeyIsFirst:
        raise capi.ThrillGpuError("InnerJoin: only the pair.first key extractors are recognised by the GPU path")
    if join_function not in (JoinKeyValues, JoinValues):
        raise capi.ThrillGpuError("InnerJoin: join function %r is not one the GPU path recognises" % (join_function,))
    if first.ctx is not second.ctx:
        raise capi.ThrillGpuError("InnerJoin: the DIAs belong to different contexts")
    for d in (first, second):
        if not (d.items.ndim == 1 and d.items.dtype == KV):
            raise capi.ThrillGpuError("InnerJoin: items must be pair<uint64_t, 8-byte value>")
    desc = capi.JoinDesc(16, join_function.code)
    sides = (capi.MergeInput * 2)()
    keep = []
    for j, d in enumerate((first, second)):
        blocks, nb = d._blocks(d.items)
        keep.append(blocks)
        sides[j].blocks = C.cast(blocks, C.POINTER(capi.Block))
        sides[j].nblocks = nb
    n_out = C.c_size_t()
    tg = first.ctx.tg
    tg.ck(tg.L.tg_inner_join_file(tg.h, C.byref(desc), C.byref(sides[0]), C.byref(sides[1]), C.byref(n_out)))
    dtype = KEY_V1_V2 if join_function is JoinKeyValues else V1_V2
    return DIA(first.ctx, first._fetch(n_out.value, dtype, dtype.itemsize, kw.get("_pinned_out")))


def _record_bytes(items, what="InnerJoin: JoinPair"):
    """item size of a DIA of records: np.void or structured items, or rows of a 2-D uint8 array"""
    if items.ndim == 1 and items.dtype.kind == "V":
        return items.dtype.itemsize
    if items.ndim == 2 and items.dtype == np.uint8:
        return items.shape[1]
    raise capi.ThrillGpuError("%s takes DIAs of np.void or structured items, not %r/%r" % (what, items.dtype, items.shape))


def _inner_join_records(first, second, key1, key2, pinned_out):
    """InnerJoin(left, right, KeyField | KeyIsFirst, KeyField | KeyIsFirst, JoinPair) on DIAs of fixed-size records: np.void
    items of left_bytes + right_bytes (tg_inner_join_records_file)"""
    keys = []
    for k in (key1, key2):
        if k is KeyIsFirst:
            keys.append((0, 8))                      # pair<uint64_t, V>: .first is the first 8 bytes
        elif getattr(k, "key_bytes", None) is not None:
            keys.append((k.key_offset, k.key_bytes))
        else:
            raise capi.ThrillGpuError("InnerJoin: JoinPair takes KeyField or pair.first key extractors, not %r" % (k,))
    if first.ctx is not second.ctx:
        raise capi.ThrillGpuError("InnerJoin: the DIAs belong to different contexts")
    lb, rb = _record_bytes(first.items), _record_bytes(second.items)
    desc = capi.JoinRecordsDesc(lb, rb, keys[0][0], keys[0][1], keys[1][0], keys[1][1])
    sides = (capi.MergeInput * 2)()
    keep = []
    for j, d in enumerate((first, second)):
        blocks, nb = d._blocks(d.items)
        keep.append(blocks)
        sides[j].blocks = C.cast(blocks, C.POINTER(capi.Block))
        sides[j].nblocks = nb
    n_out = C.c_size_t()
    tg = first.ctx.tg
    tg.ck(tg.L.tg_inner_join_records_file(tg.h, C.byref(desc), C.byref(sides[0]), C.byref(sides[1]), C.byref(n_out)))
    dtype = np.dtype((np.void, lb + rb))
    return DIA(first.ctx, first._fetch(n_out.value, dtype, lb + rb, pinned_out))


class GroupIterator(object):
    """the iterator handed to a group function (api::GroupByIterator, api/group_by_iterator.hpp:47-127): HasNext() / Next() over
    one group of the key-sorted items; Next() gives a (key, value) tuple of ints"""

    def __init__(self, items):
        self._keys, self._vals = items["key"], items["val"]
        self._pos, self._equal = 0, True
        self._key = int(self._keys[0])

    def HasNext(self):
        return self._pos < len(self._keys) and self._equal

    def Next(self):
        k, v = int(self._keys[self._pos]), int(self._vals[self._pos])
        self._pos += 1
        if self._pos < len(self._keys) and int(self._keys[self._pos]) != self._key:
            self._key = int(self._keys[self._pos])
            self._equal = False
        return k, v

    def _has_next_for_real(self):
        return self._pos < len(self._keys)

    def _get_next_key(self):
        self._equal = True
        return self._key


class DIA(object):
    def __init__(self, ctx, items):
        self.ctx = ctx
        self.items = np.ascontiguousarray(items)

    # ---- Block views of the local File ----------------------------------------------------------------
    def _blocks(self, arr, mutable=False):
        raw = arr.view(np.uint8).reshape(-1)
        n = len(raw)
        nb = (n + BLOCK_BYTES - 1) // BLOCK_BYTES
        blocks = (capi.Block * max(nb, 1))()
        for i in range(nb):
            lo = i * BLOCK_BYTES
            blocks[i].data = raw.ctypes.data + lo
            blocks[i].bytes = min(n, lo + BLOCK_BYTES) - lo
        return blocks, nb

    def _fetch(self, n_items, dtype, item_bytes, pinned_out=None):
        nbytes = n_items * item_bytes
        out = pinned_out if pinned_out is not None else np.empty(nbytes, dtype=np.uint8)
        out = out[:nbytes]
        blocks, nb = self._blocks(out)
        self.ctx.tg.ck(self.ctx.tg.L.tg_fetch_output(self.ctx.tg.h, blocks, nb))
        if dtype is None:
            return out.reshape(n_items, item_bytes)
        return out.view(dtype)

    # ---- DIA<T>::Sort ----------------------------------------------------------------------------------
    def _key_desc(self, compare_function):
        if compare_function not in (None, Less, Greater):
            raise capi.ThrillGpuError("Sort: comparator %r is not one the GPU path recognises "
                                      "(std::less / std::greater on the key)" % (compare_function,))
        desc = 1 if compare_function is Greater else 0
        it = self.items
        if it.ndim == 1 and it.dtype == np.uint64:
            return capi.KeyDesc(8, 0, 8, capi.KEY_UINT_LE, desc, 0), np.uint64
        if it.ndim == 1 and it.dtype == KV:
            return capi.KeyDesc(16, 0, 8, capi.KEY_UINT_LE, desc, 0), KV
        if it.ndim == 2 and it.dtype == np.uint8 and it.shape[1] == 100 and not desc:
            # TeraSort Record{uint8 key[10]; uint8 value[90]}, operator< = lexicographic on the key
            # (examples/terasort/terasort.cpp:31-42)
            return capi.KeyDesc(100, 0, 10, capi.KEY_BYTES_BE, 0, 0), None
        raise capi.ThrillGpuError("Sort: item type %r/%r is not supported by the GPU path" % (it.dtype, it.shape))

    def Sort(self, compare_function=None, _pinned_out=None):
        desc, dtype = self._key_desc(compare_function)
        blocks, nb = self._blocks(self.items)
        n_out = C.c_size_t()
        tg = self.ctx.tg
        tg.ck(tg.L.tg_sort_file(tg.h, C.byref(desc), blocks, nb, self.ctx._next_seed(), C.byref(n_out)))
        return DIA(self.ctx, self._fetch(n_out.value, dtype, desc.item_bytes, _pinned_out))

    # ---- DIA<T>::Merge (api/merge.hpp:715-721) ---------------------------------------------------------
    def Merge(self, second_dia, compare_function=None, _pinned_out=None):
        """merge with another DIA sorted by the same comparator; equal items come out in (input, position) order"""
        return Merge(compare_function, self, second_dia, _pinned_out=_pinned_out)

    def SortStable(self, compare_function=None):
        return self.Sort(compare_function)         # the GPU path is stable by construction

    # ---- DIA<T>::ReducePair / ReduceByKey --------------------------------------------------------------
    def ReducePair(self, reduce_function, _pinned_out=None):
        if not isinstance(reduce_function, _Functor) or reduce_function.code is None:
            raise capi.ThrillGpuError("ReducePair: reduce function %r is not one the GPU path recognises" % (reduce_function,))
        if not (self.items.ndim == 1 and self.items.dtype == KV):
            raise capi.ThrillGpuError("ReducePair: items must be pair<uint64_t, 8-byte value>")
        desc = capi.KVDesc(16, reduce_function.code)
        blocks, nb = self._blocks(self.items)
        n_out = C.c_size_t()
        tg = self.ctx.tg
        tg.ck(tg.L.tg_reduce_file(tg.h, C.byref(desc), blocks, nb, C.byref(n_out)))
        return DIA(self.ctx, self._fetch(n_out.value, KV, 16, _pinned_out))

    # ---- DIA<T>::ReduceToIndex (api/reduce_to_index.hpp:60-237) -------------------------------------------------------
    def ReduceToIndex(self, key_extractor, reduce_function, size, neutral_element=(0, 0), _pinned_out=None):
        """items: pair<uint64_t index, 8-byte value>; result: this worker's contiguous slice of the dense array of `size`
        16-byte items ((i, reduced value), or the neutral element where no item has index i); .index_begin = first index"""
        if key_extractor is not KeyIsFirst:
            raise capi.ThrillGpuError("ReduceToIndex: only the pair.first key extractor is recognised by the GPU path")
        if not isinstance(reduce_function, _Functor) or reduce_function.code is None:
            raise capi.ThrillGpuError("ReduceToIndex: reduce function %r is not one the GPU path recognises" % (reduce_function,))
        if not (self.items.ndim == 1 and self.items.dtype == KV):
            raise capi.ThrillGpuError("ReduceToIndex: items must be pair<uint64_t, 8-byte value>")
        desc = capi.KVDesc(16, reduce_function.code)
        blocks, nb = self._blocks(self.items)
        neutral = np.zeros(1, dtype=KV)
        neutral["key"], neutral["val"] = int(neutral_element[0]), int(neutral_element[1])
        n_out, begin = C.c_size_t(), C.c_uint64()
        tg = self.ctx.tg
        tg.ck(tg.L.tg_reduce_to_index_file(tg.h, C.byref(desc), blocks, nb, int(size), neutral.ctypes.data,
                                           C.byref(n_out), C.byref(begin)))
        out = DIA(self.ctx, self._fetch(n_out.value, KV, 16, _pinned_out))
        out.index_begin = int(begin.value)
        return out

    # ---- DIA<T>::GroupByKey / GroupToIndex (api/group_by_key.hpp:419-428, api/group_to_index.hpp:257-290) -------------------
    def _group(self, what, key_extractor, size=None):
        if key_extractor is not KeyIsFirst:
            raise capi.ThrillGpuError("%s: only the pair.first key extractor is recognised by the GPU path" % what)
        if not (self.items.ndim == 1 and self.items.dtype == KV):
            raise capi.ThrillGpuError("%s: items must be pair<uint64_t, 8-byte value>" % what)
        blocks, nb = self._blocks(self.items)
        inp = capi.MergeInput(None, C.cast(blocks, C.POINTER(capi.Block)), nb)
        n_out, begin, end = C.c_size_t(), C.c_uint64(), C.c_uint64()
        tg = self.ctx.tg
        if size is None:
            tg.ck(tg.L.tg_group_by_key_file(tg.h, C.byref(inp), C.byref(n_out)))
        else:
            tg.ck(tg.L.tg_group_to_index_file(tg.h, C.byref(inp), int(size), C.byref(n_out), C.byref(begin), C.byref(end)))
        return self._fetch(n_out.value, KV, 16), int(begin.value), int(end.value)

    def GroupByKey(self, key_extractor, group_function, dtype):
        """items: pair<uint64_t, 8-byte value>; group_function(iterator, key) is called once per group of this worker's share
        (worker key % p owns a key) in ascending key order, with an iterator that has HasNext() and Next() over the group's
        items in global input order; a function that stops early is called again with the rest of its group.  The result
        holds what it returns, as an array of `dtype`."""
        grouped, _, _ = self._group("GroupByKey", key_extractor)
        out = []
        if len(grouped):
            it = GroupIterator(grouped)
            while it._has_next_for_real():
                out.append(group_function(it, it._get_next_key()))
        return DIA(self.ctx, np.array(out, dtype=dtype))

    def GroupToIndex(self, key_extractor, group_function, size, neutral_element, dtype):
        """items: pair<uint64_t index, 8-byte value>; one result per index of this worker's range
        Range(0, size).Partition(rank, p): group_function(iterator, index) where the index has items, neutral_element where it
        has none.  An index >= size raises.  .index_begin = first index of the range."""
        grouped, begin, end = self._group("GroupToIndex", key_extractor, size)
        out = []
        curr = begin
        if len(grouped):
            it = GroupIterator(grouped)
            while it._has_next_for_real():
                if it._get_next_key() != curr:
                    out.append(neutral_element)
                else:
                    out.append(group_function(it, it._get_next_key()))
                curr += 1
        out.extend([neutral_element] * (end - curr))
        res = DIA(self.ctx, np.array(out, dtype=dtype))
        res.index_begin = begin
        return res

    # ---- DIA<T>::PrefixSum / ExPrefixSum (api/prefix_sum.hpp:28-128) -------------------------------------------------------
    def _scan_desc(self, what, sum_function):
        it = self.items
        if it.ndim == 1 and it.dtype == KV:
            if sum_function is None or not getattr(sum_function, "on_second", False):
                raise capi.ThrillGpuError("%s: pair items take ScanSecond(F) as the sum function" % what)
            return capi.ScanDesc(16, sum_function.code)
        if it.ndim == 1 and it.dtype == np.uint64:
            fn = PlusU64 if sum_function is None else sum_function
            if fn in (PlusU64, MinU64, MaxU64):
                return capi.ScanDesc(8, fn.code)
        if it.ndim == 1 and it.dtype == np.float64:
            fn = PlusDouble if sum_function is None else sum_function
            if fn is PlusDouble:
                return capi.ScanDesc(8, fn.code)
        raise capi.ThrillGpuError("%s: sum function %r on %r items is not one the GPU path recognises" % (what, sum_function, it.dtype))

    def _prefix_sum(self, what, sum_function, initial_element, inclusive):
        desc = self._scan_desc(what, sum_function)
        if desc.item_bytes == 16:
            ini = np.array(initial_element if initial_element is not None else (0, 0), np.uint64)
        else:
            ini = np.zeros(1, self.items.dtype)
            if initial_element is not None:
                ini[0] = initial_element
        blocks, nb = self._blocks(self.items)
        inp = capi.MergeInput(None, C.cast(blocks, C.POINTER(capi.Block)), nb)
        n_out = C.c_size_t()
        tg = self.ctx.tg
        tg.ck(tg.L.tg_prefix_sum_file(tg.h, C.byref(desc), C.byref(inp), ini.ctypes.data, int(inclusive), C.byref(n_out)))
        return DIA(self.ctx, self._fetch(n_out.value, self.items.dtype, desc.item_bytes))

    def PrefixSum(self, sum_function=None, initial_element=None):
        """out_i = carry + x_0 + ... + x_i on every worker, carry = initial_element + the local totals of the workers below
        (each folded from T()).  uint64 items with PlusU64 (the default), MinU64 or MaxU64; float64 items with PlusDouble; KV
        items with ScanSecond(F), initial_element a (first, second) tuple"""
        return self._prefix_sum("PrefixSum", sum_function, initial_element, True)

    def ExPrefixSum(self, sum_function=None, initial_element=None):
        """out_0 = carry, out_i = carry + x_0 + ... + x_{i-1}; otherwise as PrefixSum"""
        return self._prefix_sum("ExPrefixSum", sum_function, initial_element, False)

    # ---- DIA<T>::ZipWithIndex (api/zip_with_index.hpp:40-152) -------------------------------------------------------------------
    def ZipWithIndex(self, zip_function):
        """8-byte items -> KV items: (global index, item bits) with IndexFirst, (item bits, global index) with IndexSecond"""
        if zip_function not in (IndexFirst, IndexSecond):
            raise capi.ThrillGpuError("ZipWithIndex: zip function %r is not one the GPU path recognises" % (zip_function,))
        if not (self.items.ndim == 1 and self.items.dtype.itemsize == 8):
            raise capi.ThrillGpuError("ZipWithIndex: items must be 8 bytes")
        blocks, nb = self._blocks(self.items)
        inp = capi.MergeInput(None, C.cast(blocks, C.POINTER(capi.Block)), nb)
        n_out = C.c_size_t()
        tg = self.ctx.tg
        tg.ck(tg.L.tg_zip_with_index_file(tg.h, C.byref(inp), int(zip_function is IndexFirst), C.byref(n_out)))
        return DIA(self.ctx, self._fetch(n_out.value, KV, 16))

    def ReduceByKey(self, key_extractor, reduce_function, _pinned_out=None):
        """pair<uint64_t, 8-byte value> items with KeyIsFirst and a ReducePair function; or fixed-size records (np.void or structured
        items, or rows of a 2-D uint8 array: 4..1024 bytes in multiples of 4) with KeyField(offset, nbytes) (KeyIsFirst for pair items)
        and FieldReduce(runs).  Records: worker Hash128to64(0, key) % p holds a key's result, in ascending key order."""
        if getattr(reduce_function, "runs", None) is not None:
            return self._reduce_records(key_extractor, reduce_function, _pinned_out)
        if key_extractor is not KeyIsFirst:
            raise capi.ThrillGpuError("ReduceByKey: only the pair.first key extractor is recognised by the GPU path")
        return self.ReducePair(reduce_function)

    def _reduce_records(self, key_extractor, reduce_function, pinned_out):
        if key_extractor is KeyIsFirst:
            key = (0, 8)                                 # pair<uint64_t, V>: .first is the first 8 bytes
        elif getattr(key_extractor, "key_bytes", None) is not None:
            key = (key_extractor.key_offset, key_extractor.key_bytes)
        else:
            raise capi.ThrillGpuError("ReduceByKey: FieldReduce takes KeyField or pair.first key extractors, not %r" % (key_extractor,))
        it = self.items
        ib = _record_bytes(it, "ReduceByKey: FieldReduce")
        if len(reduce_function.runs) > 8:
            raise capi.ThrillGpuError("ReduceByKey: at most 8 field runs")
        desc = capi.reduce_records_desc(ib, key[0], key[1], reduce_function.runs)
        blocks, nb = self._blocks(it)
        inp = capi.MergeInput(None, C.cast(blocks, C.POINTER(capi.Block)), nb)
        n_out = C.c_size_t()
        tg = self.ctx.tg
        tg.ck(tg.L.tg_reduce_by_key_records_file(tg.h, C.byref(desc), C.byref(inp), C.byref(n_out)))
        out = self._fetch(n_out.value, None if it.ndim == 2 else it.dtype, ib, pinned_out)
        return DIA(self.ctx, out)

    # ---- actions ---------------------------------------------------------------------------------------
    def _action_desc(self, what, fn):
        it = self.items
        if it.ndim == 1 and it.dtype == KV:
            if not getattr(fn, "on_second", False):
                raise capi.ThrillGpuError("%s: pair items take ScanSecond(F) as the function" % what)
            return capi.ScanDesc(16, fn.code)
        if it.ndim == 1 and it.dtype == np.uint64 and fn in (PlusU64, MinU64, MaxU64):
            return capi.ScanDesc(8, fn.code)
        if it.ndim == 1 and it.dtype == np.float64 and fn in (PlusDouble, MinDouble, MaxDouble):
            return capi.ScanDesc(8, fn.code)
        raise capi.ThrillGpuError("%s: function %r on %r items is not one the GPU path recognises" % (what, fn, it.dtype))

    def AllReduce(self, reduce_function, initial_value=None):
        """DIA<T>::AllReduce(fn[, initial]) (api/all_reduce.hpp): the fold of every worker's items from its first one (worker 0
        from initial_value, if given; an empty worker contributes T(), or initial_value if given), then of the workers' values in
        rank order; the same value on every worker.  uint64 items with PlusU64, MinU64 or MaxU64; float64 items with PlusDouble,
        MinDouble or MaxDouble; KV items with ScanSecond(F) (any of these F), initial_value a (first, second) tuple and the
        result a (first, second) tuple of words"""
        desc = self._action_desc("AllReduce", reduce_function)
        ini = None
        if initial_value is not None:
            ini = np.array(initial_value, np.uint64) if desc.item_bytes == 16 else np.array([initial_value], self.items.dtype)
        out = np.zeros(2 if desc.item_bytes == 16 else 1, np.uint64 if desc.item_bytes == 16 else self.items.dtype)
        blocks, nb = self._blocks(self.items)
        inp = capi.MergeInput(None, C.cast(blocks, C.POINTER(capi.Block)), nb)
        tg = self.ctx.tg
        tg.ck(tg.L.tg_all_reduce_file(tg.h, C.byref(desc), C.byref(inp), None if ini is None else ini.ctypes.data,
                                      out.ctypes.data))
        return (int(out[0]), int(out[1])) if desc.item_bytes == 16 else out[0]

    def Sum(self, sum_function=None, initial_value=None):
        """DIA<T>::Sum (api/sum.hpp): AllReduce with PlusU64 / PlusDouble by default"""
        if sum_function is None:
            sum_function = PlusDouble if self.items.dtype == np.float64 else PlusU64
        return self.AllReduce(sum_function, initial_value)

    def Min(self, initial_value=None):
        """DIA<T>::Min (api/min.hpp): AllReduce with common::minimum, std::min(a, b) = b < a ? b : a"""
        return self.AllReduce(MinDouble if self.items.dtype == np.float64 else MinU64, initial_value)

    def Max(self, initial_value=None):
        """DIA<T>::Max (api/max.hpp): AllReduce with common::maximum, std::max(a, b) = a < b ? b : a"""
        return self.AllReduce(MaxDouble if self.items.dtype == np.float64 else MaxU64, initial_value)

    def HyperLogLog(self, precision):
        """The registers of DIA<T>::HyperLogLog<p> (api/hyperloglog.hpp): SipHash-2-4 of every item into 2^precision one-byte
        registers, merged over the workers by max; a uint8 array, the same on every worker.  uint64, float64 (hashed as bits)
        and KV items.  The estimate is the stock HyperLogLogRegisters<p>::result()'s to compute, not this mirror's."""
        it = self.items
        if it.ndim != 1 or it.dtype not in (np.uint64, np.float64, KV):
            raise capi.ThrillGpuError("HyperLogLog: %r items are not ones the GPU path recognises" % (it.dtype,))
        if not 4 <= precision <= 18:
            raise capi.ThrillGpuError("HyperLogLog: precision %r is outside 4..18" % (precision,))
        out = np.zeros(1 << precision, np.uint8)
        blocks, nb = self._blocks(it)
        inp = capi.MergeInput(None, C.cast(blocks, C.POINTER(capi.Block)), nb)
        tg = self.ctx.tg
        tg.ck(tg.L.tg_hyperloglog_file(tg.h, it.dtype.itemsize, precision, C.byref(inp), out.ctypes.data))
        return out

    # ---- DIA<T>::Window (api/window.hpp:284-380, :524-564) -----------------------------------------------------------------------
    def Window(self, window_size, fn, partial=False, disjoint=False):
        """The left fold with fn of every window of window_size consecutive items, on the worker that holds the window's last
        item (thrill_gpu::Window with WindowFold<F>).  partial: the last worker also emits the folds of the last min(N, k-1)
        suffixes (Window(k, f, partial_f)).  disjoint: the windows [jk, jk+k-1], the trailing N mod k items folded on the last
        worker (Window(DisjointTag, k, f)).  The items and functions are those of AllReduce; window_size is 2..4096."""
        if partial and disjoint:
            raise capi.ThrillGpuError("Window: a disjoint Window has no partial function")
        desc = self._action_desc("Window", fn)
        mode = capi.WINDOW_DISJOINT if disjoint else capi.WINDOW_PARTIAL if partial else capi.WINDOW_FULL
        blocks, nb = self._blocks(self.items)
        inp = capi.MergeInput(None, C.cast(blocks, C.POINTER(capi.Block)), nb)
        n_out = C.c_size_t()
        tg = self.ctx.tg
        tg.ck(tg.L.tg_window_file(tg.h, C.byref(desc), C.byref(inp), int(window_size), mode, C.byref(n_out)))
        return DIA(self.ctx, self._fetch(n_out.value, self.items.dtype, desc.item_bytes))

    # ---- DIA<T>::Sample / BernoulliSample (api/sample.hpp:37-140, api/bernoulli_sample.hpp:27-77) ----------------------------------
    def _sample(self, what, call, param, seed):
        it = self.items
        ib = it.dtype.itemsize * (it.shape[1] if it.ndim == 2 else 1)
        if it.ndim not in (1, 2) or ib % 4 or not 4 <= ib <= 256:
            raise capi.ThrillGpuError("%s: %d-byte items (a multiple of 4 bytes from 4 to 256)" % (what, ib))
        seed = self.ctx._next_seed() if seed is None else int(seed) % (1 << 64)
        blocks, nb = self._blocks(it)
        inp = capi.MergeInput(None, C.cast(blocks, C.POINTER(capi.Block)), nb)
        n_out = C.c_size_t()
        tg = self.ctx.tg
        tg.ck(call(tg.h, ib, C.byref(inp), param, seed, C.byref(n_out)))
        out = self._fetch(n_out.value, None if it.ndim == 2 else it.dtype, ib)
        return DIA(self.ctx, out.view(it.dtype) if it.ndim == 2 else out)

    def Sample(self, sample_size, seed=None):
        """A uniform sample of min(sample_size, N) items without replacement: the positions with the sample_size smallest keys
        key(seed, g) (include/thrill_gpu.h), each kept item on its worker in input order.  Rank 0's seed wins; without one every
        rank draws ctx._next_seed()."""
        return self._sample("Sample", self.ctx.tg.L.tg_sample_file, int(sample_size), seed)

    def BernoulliSample(self, p, seed=None):
        """Every item kept independently with probability p: position g iff (key(seed, g) >> 11) < ceil(p * 2^53), kept items on
        their worker in input order.  p outside [0, 1] or NaN is an error."""
        return self._sample("BernoulliSample", self.ctx.tg.L.tg_bernoulli_sample_file, float(p), seed)

    def Size(self):
        n = len(self.items)
        if self.ctx.num_workers() > 1:
            import torch
            import torch.distributed as dist
            t = torch.tensor([n], dtype=torch.int64)
            dist.all_reduce(t)
            n = int(t.item())
        return n

    def AllGather(self):
        if self.ctx.num_workers() == 1:
            return self.items
        import torch.distributed as dist
        parts = [None] * self.ctx.num_workers()
        dist.all_gather_object(parts, self.items)
        return np.concatenate(parts)

    def Gather(self, root=0):
        allv = self.AllGather()
        return allv if self.ctx.my_rank() == root else allv[:0]
