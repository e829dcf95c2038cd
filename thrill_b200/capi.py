"""ctypes binding of the C ABI in include/thrill_gpu.h (libthrill_gpu.so, hand-written sm_90a CUDA).

Fails loudly when the shared library is missing or no H100 is present — there is no CPU fallback and
nothing here ever touches oracle/.
"""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("TG_LIB") or os.path.join(HERE, "csrc", "libthrill_gpu.so")      # TG_LIB: another build of the library, e.g. for an A/B comparison

TG_OK = 0
KEY_UINT_LE, KEY_BYTES_BE = 0, 1
OP_SUM_F64, OP_SUM_U64, OP_MIN_U64, OP_MAX_U64, OP_MIN_F64, OP_MAX_F64, OP_FIRST = range(7)
K_RADIX_HIST, K_PARTITION, K_MERGE, K_PREAGG, K_AGGREGATE, K_COMPACT, K_OTHER, K_FIXUP, K_SEGCOUNT, K_EXCHANGE, K_JOIN, K_SCAN = \
    range(12)
JOIN_KEY_VALUES, JOIN_VALUES = 0, 1


class KeyDesc(C.Structure):
    _fields_ = [("item_bytes", C.c_uint32), ("key_offset", C.c_uint32), ("key_bytes", C.c_uint32),
                ("key_kind", C.c_uint32), ("descending", C.c_uint32), ("stable", C.c_uint32)]


class KVDesc(C.Structure):
    _fields_ = [("item_bytes", C.c_uint32), ("op", C.c_uint32)]


class Block(C.Structure):
    _fields_ = [("data", C.c_void_p), ("bytes", C.c_size_t)]


class DevFile(C.Structure):
    _fields_ = [("dptr", C.c_void_p), ("items", C.c_uint64), ("item_bytes", C.c_uint32), ("reserved", C.c_uint32)]


class MergeInput(C.Structure):
    """tg_merge_input: a device File (dev) or a host File (blocks, nblocks)"""
    _fields_ = [("dev", C.POINTER(DevFile)), ("blocks", C.POINTER(Block)), ("nblocks", C.c_size_t)]


class JoinDesc(C.Structure):
    _fields_ = [("item_bytes", C.c_uint32), ("join_fn", C.c_uint32)]


class ScanDesc(C.Structure):
    _fields_ = [("item_bytes", C.c_uint32), ("op", C.c_uint32)]


class BlockGeom(C.Structure):
    _fields_ = [("bytes", C.c_uint64), ("first_item", C.c_uint64), ("num_items", C.c_uint64)]


def u64_desc(descending=False):
    return KeyDesc(8, 0, 8, KEY_UINT_LE, int(descending), 0)


def kv_key_desc():
    return KeyDesc(16, 0, 8, KEY_UINT_LE, 0, 0)


def record_desc():
    return KeyDesc(100, 0, 10, KEY_BYTES_BE, 0, 0)


# every symbol include/thrill_gpu.h declares: (name, restype, argtypes)
_vp, _u64, _sz, _i, _u32 = C.c_void_p, C.c_uint64, C.c_size_t, C.c_int, C.c_uint32
_P = C.POINTER
SYMBOLS = [
    ("tg_version", _i, []),
    ("tg_device_count", _i, []),
    ("tg_strerror", C.c_char_p, [_i]),
    ("tg_last_error", C.c_char_p, [_vp]),
    ("tg_get_unique_id", _i, [_vp]),
    ("tg_init", _i, [_i, _i, _i, _vp, _P(_vp)]),
    ("tg_shutdown", _i, [_vp]),
    ("tg_rank", _i, [_vp]),
    ("tg_nranks", _i, [_vp]),
    ("tg_stream", _vp, [_vp]),
    ("tg_sync", _i, [_vp]),
    ("tg_barrier", _i, [_vp]),
    ("tg_alloc", _i, [_vp, _sz, _P(_vp)]),
    ("tg_free", _i, [_vp, _vp]),
    ("tg_timer_start", _i, [_vp]),
    ("tg_timer_stop", _i, [_vp, _P(C.c_float)]),
    ("tg_launch_count", _u64, [_vp]),
    ("tg_prefix_sort_fallbacks", _u64, [_vp]),
    ("tg_hot_records", _u64, [_vp]),
    ("tg_profile_enable", _i, [_vp, _i]),
    ("tg_profile_get", _i, [_vp, _i, _P(C.c_float), _P(_u64)]),
    ("tg_profile_list", _i, [_vp, _i, _P(C.c_float), _sz, _P(_sz)]),
    ("tg_host_alloc", _i, [_vp, _sz, _P(_vp)]),
    ("tg_host_free", _i, [_vp, _vp]),
    ("tg_upload", _i, [_vp, _vp, _vp, _sz]),
    ("tg_download", _i, [_vp, _vp, _vp, _sz]),
    ("tg_upload_blocks", _i, [_vp, _vp, _P(Block), _sz, _P(_sz)]),
    ("tg_download_blocks", _i, [_vp, _vp, _P(Block), _sz]),
    ("tg_file_geometry", _sz, [_u64, _u32, _u64, _u64, _P(BlockGeom), _sz]),
    ("tg_radix_sort_local", _i, [_vp, _P(KeyDesc), _vp, _vp, _sz]),
    ("tg_sample_size", _u64, [_u64]),
    ("tg_select_splitters", _i, [_P(KeyDesc), _vp, _u64, _u32, _vp]),
    ("tg_draw_samples", _i, [_vp, _P(KeyDesc), _vp, _sz, _u64, _u64, _vp, _P(_u64)]),
    ("tg_classify_scatter", _i, [_vp, _P(KeyDesc), _vp, _sz, _u64, _vp, _u32, _vp, _P(_u64)]),
    ("tg_sort_select", _i, [_vp, _P(KeyDesc), _P(_vp), _P(_sz), _u32, _u64, _vp, _P(_vp), _P(_u64), _P(_u64)]),
    ("tg_kway_merge", _i, [_vp, _P(KeyDesc), _vp, _P(_u64), _u32, _vp, _vp]),
    ("tg_hash_aggregate", _i, [_vp, _P(KVDesc), _vp, _sz, _vp, _P(_u64)]),
    ("tg_hash_partition", _i, [_vp, _P(KVDesc), _vp, _sz, _u32, _vp, _P(_u64)]),
    ("tg_range_partition", _i, [_vp, _vp, _sz, _u64, _u32, _vp, _P(_u64)]),
    ("tg_exchange_plan", _i, [_u32, _u32, _P(_u32), _P(_u64), _P(_u64), _P(_u64), _P(_u64), _P(_u64)]),
    ("tg_sort", _i, [_vp, _P(KeyDesc), _vp, _sz, _u64, _P(_vp), _P(_sz)]),
    ("tg_reduce_by_key", _i, [_vp, _P(KVDesc), _vp, _sz, _P(_vp), _P(_sz)]),
    ("tg_reduce_to_index", _i, [_vp, _P(KVDesc), _vp, _sz, _u64, _vp, _P(_vp), _P(_sz), _P(_u64)]),
    ("tg_reduce_to_index_file", _i, [_vp, _P(KVDesc), _P(Block), _sz, _u64, _vp, _P(_sz), _P(_u64)]),
    ("tg_sort_file", _i, [_vp, _P(KeyDesc), _P(Block), _sz, _u64, _P(_sz)]),
    ("tg_reduce_file", _i, [_vp, _P(KVDesc), _P(Block), _sz, _P(_sz)]),
    ("tg_fetch_output", _i, [_vp, _P(Block), _sz]),
    ("tg_output_detach", _i, [_vp, _P(DevFile)]),
    ("tg_dev_file_fetch", _i, [_vp, _P(DevFile), _P(Block), _sz]),
    ("tg_dev_file_free", _i, [_vp, _P(DevFile)]),
    ("tg_sort_dev", _i, [_vp, _P(KeyDesc), _P(DevFile), _u64, _P(_sz)]),
    ("tg_reduce_dev", _i, [_vp, _P(KVDesc), _P(DevFile), _P(_sz)]),
    ("tg_reduce_to_index_dev", _i, [_vp, _P(KVDesc), _P(DevFile), _u64, _vp, _P(_sz), _P(_u64)]),
    ("tg_merge", _i, [_vp, _P(KeyDesc), _P(_vp), _P(_sz), _u32, _P(_vp), _P(_sz)]),
    ("tg_merge_file", _i, [_vp, _P(KeyDesc), _P(MergeInput), _u32, _P(_sz)]),
    ("tg_merge_select", _i, [_vp, _P(KeyDesc), _P(_vp), _P(_sz), _u32, _u32, _P(_u64)]),
    ("tg_merge_plan", _i, [_u32, _u32, _P(_u64), _P(_u64), _P(_u64), _P(_u64)]),
    ("tg_inner_join", _i, [_vp, _P(JoinDesc), _vp, _sz, _vp, _sz, _P(_vp), _P(_sz)]),
    ("tg_inner_join_file", _i, [_vp, _P(JoinDesc), _P(MergeInput), _P(MergeInput), _P(_sz)]),
    ("tg_group_by_key", _i, [_vp, _vp, _sz, _P(_vp), _P(_sz)]),
    ("tg_group_to_index", _i, [_vp, _vp, _sz, _u64, _P(_vp), _P(_sz), _P(_u64), _P(_u64)]),
    ("tg_group_by_key_file", _i, [_vp, _P(MergeInput), _P(_sz)]),
    ("tg_group_to_index_file", _i, [_vp, _P(MergeInput), _u64, _P(_sz), _P(_u64), _P(_u64)]),
    ("tg_mod_partition", _i, [_vp, _vp, _sz, _u32, _vp, _P(_u64)]),
    ("tg_prefix_sum", _i, [_vp, _P(ScanDesc), _vp, _sz, _vp, _i, _P(_vp), _P(_sz)]),
    ("tg_zip_with_index", _i, [_vp, _vp, _sz, _i, _P(_vp), _P(_sz)]),
    ("tg_prefix_sum_file", _i, [_vp, _P(ScanDesc), _P(MergeInput), _vp, _i, _P(_sz)]),
    ("tg_zip_with_index_file", _i, [_vp, _P(MergeInput), _i, _P(_sz)]),
    ("tg_scan_local_total", _i, [_vp, _P(ScanDesc), _vp, _sz, _vp]),
    ("tg_prefix_sum_select", _i, [_vp, _P(ScanDesc), _vp, _sz, _u32, _u32, _vp, _vp, _i, _P(_vp), _P(_sz)]),
    ("tg_zip_with_index_select", _i, [_vp, _vp, _sz, _u32, _u32, _P(_u64), _i, _P(_vp), _P(_sz)]),
    ("tg_all_reduce", _i, [_vp, _P(ScanDesc), _vp, _sz, _vp, _vp]),
    ("tg_all_reduce_file", _i, [_vp, _P(ScanDesc), _P(MergeInput), _vp, _vp]),
    ("tg_all_reduce_select", _i, [_vp, _P(ScanDesc), _P(_vp), _P(_sz), _u32, _vp, _vp]),
    ("tg_transfer_bytes", _i, [_vp, _P(_u64), _P(_u64)]),
    ("tg_gen_sort_uniform", _i, [_vp, _vp, _u64, _u64, _u64]),
    ("tg_gen_reduce_uniform", _i, [_vp, _vp, _u64, _u64, _u64, _u64, _i]),
    ("tg_gen_sort_zipf", _i, [_vp, _vp, _u64, _u64, _u64, _vp, _u64]),
    ("tg_gen_reduce_zipf", _i, [_vp, _vp, _u64, _u64, _u64, _vp, _u64, _i]),
    ("tg_gen_records", _i, [_vp, _vp, _u64, _u64, _u64]),
    ("tg_checksum", _i, [_vp, _vp, _sz, _u32, _P(_u64)]),
    ("tg_is_sorted", _i, [_vp, _P(KeyDesc), _vp, _sz, _P(_u64)]),
]

_lib = None


class ThrillGpuError(RuntimeError):
    pass


def _preload_nccl():
    """libthrill_gpu.so needs libnccl.so.2.  If PyTorch is (or will be) in the process, its bundled NCCL must
    be the one the loader binds to that SONAME — an older system libnccl loaded first breaks `import torch`."""
    import importlib.util
    try:
        spec = importlib.util.find_spec("nvidia.nccl")
    except (ImportError, ValueError):
        spec = None
    if spec and spec.submodule_search_locations:
        for d in spec.submodule_search_locations:
            cand = os.path.join(d, "lib", "libnccl.so.2")
            if os.path.exists(cand):
                C.CDLL(cand, mode=C.RTLD_GLOBAL)
                return


def lib():
    """Load libthrill_gpu.so.  Raises if it has not been built: the product path never falls back."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ThrillGpuError("libthrill_gpu.so is not built (%s): run `python -c 'import __graft_entry__ as g; "
                                 "g.build()'` or `make -C thrill_b200/csrc`" % LIB_PATH)
        _preload_nccl()
        L = C.CDLL(LIB_PATH)
        for name, res, args in SYMBOLS:
            fn = getattr(L, name)      # AttributeError if the library does not export a declared symbol
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(status, ctx=None):
    if status != TG_OK:
        L = lib()
        msg = L.tg_strerror(status).decode()
        if ctx:
            msg += ": " + L.tg_last_error(ctx).decode()
        raise ThrillGpuError("libthrill_gpu: %s (status %d)" % (msg, status))


class Ctx(object):
    """One tg_ctx: one worker thread / GPU / stream / NCCL rank."""

    def __init__(self, device=0, rank=0, nranks=1, unique_id=None):
        import numpy as np
        self.np = np
        self.L = lib()
        self.h = C.c_void_p()
        uid = None
        if nranks > 1:
            assert unique_id is not None and len(unique_id) == 128
            uid = C.create_string_buffer(bytes(unique_id), 128)
        st = self.L.tg_init(device, rank, nranks, uid, C.byref(self.h))
        if st != TG_OK:
            raise ThrillGpuError("tg_init failed: %s%s" % (
                self.L.tg_strerror(st).decode(),
                (": " + self.L.tg_last_error(self.h).decode()) if self.h else ""))
        self.rank, self.nranks, self.device = rank, nranks, device

    def close(self):
        if self.h:
            self.L.tg_shutdown(self.h)
            self.h = C.c_void_p()

    def ck(self, st):
        check(st, self.h)

    # -- memory
    def alloc(self, nbytes):
        p = C.c_void_p()
        self.ck(self.L.tg_alloc(self.h, nbytes, C.byref(p)))
        return p.value

    def free(self, dptr):
        self.ck(self.L.tg_free(self.h, dptr))

    def upload(self, dptr, arr):
        arr = self.np.ascontiguousarray(arr)
        self.ck(self.L.tg_upload(self.h, dptr, arr.ctypes.data, arr.nbytes))
        self.sync()

    def download(self, dptr, nbytes, dtype=None):
        out = self.np.empty(nbytes, dtype=self.np.uint8)
        self.ck(self.L.tg_download(self.h, out.ctypes.data, dptr, nbytes))
        self.sync()
        return out if dtype is None else out.view(dtype)

    def to_device(self, arr):
        arr = self.np.ascontiguousarray(arr)
        d = self.alloc(max(arr.nbytes, 16))
        self.upload(d, arr)
        return d

    def sync(self):
        self.ck(self.L.tg_sync(self.h))

    def barrier(self):
        self.ck(self.L.tg_barrier(self.h))

    def timer_start(self):
        self.ck(self.L.tg_timer_start(self.h))

    def timer_stop(self):
        ms = C.c_float()
        self.ck(self.L.tg_timer_stop(self.h, C.byref(ms)))
        return ms.value

    def launches(self):
        return int(self.L.tg_launch_count(self.h))

    def profile_enable(self, on=True):
        self.ck(self.L.tg_profile_enable(self.h, int(on)))

    def profile_get(self, cls):
        ms = C.c_float(); cnt = C.c_uint64()
        self.ck(self.L.tg_profile_get(self.h, cls, C.byref(ms), C.byref(cnt)))
        return ms.value, cnt.value

    def profile_list(self, cls, cap=4096):
        buf = (C.c_float * cap)(); n = C.c_size_t()
        self.ck(self.L.tg_profile_list(self.h, cls, buf, cap, C.byref(n)))
        return [buf[i] for i in range(min(n.value, cap))]

    def host_alloc(self, nbytes):
        """page-locked host buffer as a numpy uint8 array (freed with host_free)"""
        p = C.c_void_p()
        self.ck(self.L.tg_host_alloc(self.h, max(nbytes, 16), C.byref(p)))
        arr = self.np.ctypeslib.as_array((C.c_uint8 * max(nbytes, 16)).from_address(p.value))
        arr = arr[:nbytes]
        self._pinned = getattr(self, "_pinned", {})
        self._pinned[arr.ctypes.data] = p.value
        return arr

    def host_free(self, arr):
        p = self._pinned.pop(arr.ctypes.data)
        self.ck(self.L.tg_host_free(self.h, p))

    # -- probes
    def checksum(self, dptr, n, item_bytes):
        out = (C.c_uint64 * 2)()
        self.ck(self.L.tg_checksum(self.h, dptr, n, item_bytes, out))
        return int(out[0]), int(out[1])

    def is_sorted(self, desc, dptr, n):
        v = C.c_uint64()
        self.ck(self.L.tg_is_sorted(self.h, C.byref(desc), dptr, n, C.byref(v)))
        return v.value == 0
