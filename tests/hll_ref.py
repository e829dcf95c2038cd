"""The numpy model of the HyperLogLog action (include/thrill_gpu.h, tg_hyperloglog): SipHash-2-4 with the key bytes 0..15 over
8- or 16-byte items, vectorised on uint64 arrays, and the dense register rule of the stock HyperLogLogRegisters<p>
(core/hyperloglog.cpp:1733-1740): index = h >> (64 - p), w = h << p, value = (64 - p if w == 0 else clz(w)) + 1, register = max.
Written from the SipHash specification (Aumasson and Bernstein, "SipHash: a fast short-input PRF", 2012).

Also the reader of tests/golden/reference_outputs_hll.npz (make_golden_hll.py), whose layout is:
    precisions            the p of every stored result, in the driver's order
    in_names, in_mode,    the inputs, stored once: name, mode (0 u64, 1 pair, 2 hash: words given to insert_hash directly),
    in_start, words       and their words as slices [in_start[i], in_start[i + 1]) of `words`
    in_range[i]           (start, nwords): where nwords > 0 the input is the words start, start + 1, ... and is not stored
    digest[i, k]          SHA-256 of the dense registers (a) of input i at precisions[k]
    regs_<i>_<p>          the registers (a) themselves, where they are small or mostly zero
    est_a[i, k]           the stock result() of (a)
    lay_input, lay_counts the sharded runs of the natural path: input, per-worker item counts (-1 pads to 8 workers)
    lay_dense[j, k]       1 if the natural path's sum was dense at the end, 0 if still sparse
    lay_equal[j, k]       1 if its registers (after toDense()) equal (a)
    lay_est[j, k]         its stock result()
"""
import hashlib

import numpy as np

PRECISIONS = (4, 8, 12, 14, 16, 18)
MODES = ("u64", "pair", "hash")
M64 = (1 << 64) - 1
LIMIT = 1 << 30


def _rotl(x, r):
    return (x << np.uint64(r)) | (x >> np.uint64(64 - r))


def _sipround(v0, v1, v2, v3):
    v0 = v0 + v1
    v1 = _rotl(v1, 13) ^ v0
    v0 = _rotl(v0, 32)
    v2 = v2 + v3
    v3 = _rotl(v3, 16) ^ v2
    v0 = v0 + v3
    v3 = _rotl(v3, 21) ^ v0
    v2 = v2 + v1
    v1 = _rotl(v1, 17) ^ v2
    v2 = _rotl(v2, 32)
    return v0, v1, v2, v3


def siphash24(words, item_bytes):
    """SipHash-2-4, key bytes 0, 1, ..., 15, of every item of `words` (uint64, little-endian message words; a 16-byte item is
    two consecutive words): a uint64 array"""
    words = np.ascontiguousarray(words, np.uint64).reshape(-1)
    assert item_bytes in (8, 16)
    msg = [words] if item_bytes == 8 else [words[0::2], words[1::2]]
    n = len(msg[0])
    k0, k1 = np.uint64(0x0706050403020100), np.uint64(0x0F0E0D0C0B0A0908)
    with np.errstate(over="ignore"):
        v0 = np.full(n, k0 ^ np.uint64(0x736F6D6570736575), np.uint64)
        v1 = np.full(n, k1 ^ np.uint64(0x646F72616E646F6D), np.uint64)
        v2 = np.full(n, k0 ^ np.uint64(0x6C7967656E657261), np.uint64)
        v3 = np.full(n, k1 ^ np.uint64(0x7465646279746573), np.uint64)
        # the last word holds the message length in its top byte and the (here: no) remaining bytes
        for m in msg + [np.uint64(item_bytes << 56)]:
            v3 = v3 ^ m
            v0, v1, v2, v3 = _sipround(v0, v1, v2, v3)
            v0, v1, v2, v3 = _sipround(v0, v1, v2, v3)
            v0 = v0 ^ m
        v2 = v2 ^ np.uint64(0xFF)
        for _ in range(4):
            v0, v1, v2, v3 = _sipround(v0, v1, v2, v3)
        return v0 ^ v1 ^ v2 ^ v3


def clz64(w):
    """leading zeros of every uint64 of w (64 for 0)"""
    w = np.asarray(w, np.uint64)
    n = np.zeros(w.shape, np.int64)
    x = w.copy()
    for s in (32, 16, 8, 4, 2, 1):
        top = x >> np.uint64(64 - s)
        z = top == 0
        n += np.where(z, s, 0)
        x = np.where(z, x << np.uint64(s), x)
    return np.where(w == 0, 64, n)


def index_value(hashes, p):
    """the register index and the register value of every hash"""
    h = np.asarray(hashes, np.uint64)
    w = h << np.uint64(p)
    val = np.where(w == 0, 64 - p, clz64(w)) + 1
    return (h >> np.uint64(64 - p)).astype(np.int64), val.astype(np.uint8)


def registers_from_hashes(hashes, p):
    regs = np.zeros(1 << p, np.uint8)
    idx, val = index_value(hashes, p)
    np.maximum.at(regs, idx, val)
    return regs


def registers(words, item_bytes, p):
    """the 2^p dense registers of the items"""
    return registers_from_hashes(siphash24(words, item_bytes), p)


def merge(register_sets):
    """mergeDense (core/hyperloglog.cpp:1761-1768): the per-register max"""
    out = np.array(register_sets[0], np.uint8, copy=True)
    for r in register_sets[1:]:
        np.maximum(out, r, out=out)
    return out


def digest(regs):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(regs, np.uint8).tobytes()).digest(), np.uint8)


def shards_of(words, item_bytes, counts):
    wpi = item_bytes // 8
    out, begin = [], 0
    for c in counts:
        out.append(words[begin * wpi:(begin + c) * wpi])
        begin += c
    return out


class Golden(object):
    def __init__(self, path):
        self.z = np.load(path)
        self.precisions = [int(p) for p in self.z["precisions"]]
        self.names = [str(s) for s in self.z["in_names"]]

    def mode(self, i):
        return MODES[int(self.z["in_mode"][i])]

    def item_bytes(self, i):
        return 16 if self.mode(i) == "pair" else 8

    def words(self, i):
        start, nwords = (int(x) for x in self.z["in_range"][i])
        if nwords:
            return np.uint64(start) + np.arange(nwords, dtype=np.uint64)
        s = self.z["in_start"]
        return self.z["words"][int(s[i]):int(s[i + 1])]

    def n_items(self, i):
        return len(self.words(i)) // (self.item_bytes(i) // 8)

    def digest(self, i, p):
        return self.z["digest"][i, self.precisions.index(p)]

    def regs(self, i, p):
        """the stored registers (a), or None where only their digest is kept"""
        key = "regs_%d_%d" % (i, p)
        return self.z[key] if key in self.z.files else None

    def model_registers(self, i, p):
        if self.mode(i) == "hash":
            return registers_from_hashes(self.words(i), p)
        return registers(self.words(i), self.item_bytes(i), p)

    def layouts(self, i=None):
        """(row, input, counts) of every sharded run (of input i)"""
        out = []
        for j, inp in enumerate(self.z["lay_input"]):
            if i is None or int(inp) == i:
                out.append((j, int(inp), [int(c) for c in self.z["lay_counts"][j] if c >= 0]))
        return out
