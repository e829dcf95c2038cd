"""numpy model of Sample and BernoulliSample by global position (include/thrill_gpu.h, thrill_b200/csrc/tg_sample.cu).

Position g has the key key(seed, g) = mix(mix(seed) + (g + 1) * GAMMA) mod 2^64, mix the SplitMix64 output function.
Sample(s) keeps the s positions with the smallest keys (every position if s >= N), BernoulliSample(p) keeps the positions with
(key >> 11) < ceil(p * 2^53).  Kept items stay on their worker in input order, so a worker's output is its shard masked.
"""
import math

import numpy as np

GAMMA = 0x9E3779B97F4A7C15
M64 = (1 << 64) - 1


def mix_int(z):
    """the SplitMix64 output function on a Python int (the scalar reference)"""
    z &= M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def key_int(seed, g):
    return mix_int(mix_int(seed) + (g + 1) * GAMMA)


def mix(z):
    """the same on a uint64 array (wrapping arithmetic)"""
    z = np.asarray(z, np.uint64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def keys(seed, g):
    """key(seed, g) for a uint64 array of global positions g (seed: an int, or a uint64 array broadcast against g)"""
    ms = mix(np.asarray(seed, np.uint64) if not isinstance(seed, int) else np.uint64(seed % (1 << 64)))
    g = np.asarray(g, np.uint64)
    with np.errstate(over="ignore"):
        return mix(ms + (g + np.uint64(1)) * np.uint64(GAMMA))


def bernoulli_threshold(p):
    """ceil(p * 2^53): position g is kept iff (key >> 11) < this"""
    p = float(p)
    if not 0.0 <= p <= 1.0:
        raise ValueError("BernoulliSample: probability %r outside [0, 1]" % (p,))
    return math.ceil(math.ldexp(p, 53))


def sample_mask(seed, N, s):
    """bool mask over the N global positions: the s positions with the smallest keys"""
    if s >= N:
        return np.ones(N, bool)
    if s == 0:
        return np.zeros(N, bool)
    k = keys(seed, np.arange(N, dtype=np.uint64))
    K = np.partition(k, s - 1)[s - 1]
    return k <= K


def bernoulli_mask(seed, N, p):
    t = bernoulli_threshold(p)
    if t >= 1 << 53:
        return np.ones(N, bool)
    k = keys(seed, np.arange(N, dtype=np.uint64))
    return (k >> np.uint64(11)) < np.uint64(t)


def split(items, mask, sizes):
    """each worker's output: its shard of items (sizes[w] consecutive items) where mask is set, in input order"""
    out, f = [], 0
    for n in sizes:
        out.append(items[f:f + n][mask[f:f + n]])
        f += n
    return out


def sample(shards, s, seed):
    """per-worker outputs of Sample(s) over shards (a list of arrays, worker order)"""
    sizes = [len(x) for x in shards]
    items = np.concatenate(shards) if shards else np.zeros(0)
    return split(items, sample_mask(seed, sum(sizes), s), sizes)


def bernoulli_sample(shards, p, seed):
    sizes = [len(x) for x in shards]
    items = np.concatenate(shards) if shards else np.zeros(0)
    return split(items, bernoulli_mask(seed, sum(sizes), p), sizes)


def subsets_sample(seeds, N, s):
    """for each seed (a uint64 array), the kept positions of Sample(s) of N items as a (len(seeds), s) sorted index array"""
    g = np.arange(N, dtype=np.uint64)
    k = keys(np.asarray(seeds, np.uint64)[:, None], g[None, :])
    return np.sort(np.argsort(k, axis=1)[:, :s], axis=1)
