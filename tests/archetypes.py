"""The 10 archetype container contents x 3 encodings used by the reference's TestContainerCombinations
(restated from roaring/roaring_helpers_test.go:12-232,257-305 as value sets)."""
import numpy as np

from oracle import oracle as O

W = 1 << 16


def archetype_values(name):
    if name == "empty":
        return np.zeros(0, dtype=np.int64)
    if name == "full":
        return np.arange(W)
    if name == "firstBitSet":
        return np.array([0])
    if name == "lastBitSet":
        return np.array([W - 1])
    if name == "firstBitUnset":
        return np.arange(1, W)
    if name == "lastBitUnset":
        return np.arange(0, W - 1)
    if name == "innerBitsSet":
        return np.arange(1, W - 1)
    if name == "outerBitsSet":
        return np.array([0, W - 1])
    if name == "oddBitsSet":
        return np.arange(1, W, 2)
    if name == "evenBitsSet":
        return np.arange(0, W, 2)
    raise KeyError(name)


NAMES = ["empty", "full", "firstBitSet", "lastBitSet", "firstBitUnset", "lastBitUnset", "innerBitsSet",
         "outerBitsSet", "oddBitsSet", "evenBitsSet"]


def container(name, typ):
    """explicit-encoding container, like doContainer() (roaring_helpers_test.go:246-257); note the reference's
    run archetypes for odd/even hold 32768 single-value runs"""
    return container_of(archetype_values(name), typ)


def container_of(vals, typ):
    """the sorted unique values `vals` as a container of encoding `typ` (O.ARRAY / O.BITMAP / O.RUN), whatever their number:
    to_bytes(optimize=False) keeps it as built"""
    vals = np.asarray(vals, dtype=np.int64)
    if typ == O.ARRAY:
        return O.Container.array(vals)
    if typ == O.BITMAP:
        w = np.zeros(1024, dtype=np.uint64)
        if len(vals):
            np.bitwise_or.at(w, vals >> 6, np.uint64(1) << (vals & 63).astype(np.uint64))
        return O.Container.bitmap(w)
    # runs
    if len(vals) == 0:
        return O.Container.run(np.zeros((0, 2), dtype=np.uint16))
    brk = np.nonzero(np.diff(vals) != 1)[0]
    starts = np.concatenate([[vals[0]], vals[brk + 1]])
    lasts = np.concatenate([vals[brk], [vals[-1]]])
    return O.Container.run(np.stack([starts, lasts], axis=1))


# ---------------------------------------------------------------------------------------------------
# The 20 benchmark archetypes of roaring/container_archetypes.go:19-40 (BenchmarkCtOps / TestIntersectVariants).  Their
# SHAPES are pinned by name (element / run counts, run geometry :79-121, bitmaps with exactly N bits :123-160); their
# exact contents come from a test-only RNG (molecula/apophenia, seed 23) that is not in the reference tree, so the
# contents here are drawn from numpy instead (SURVEY §8c: contents unpinned, properties pinned).
# ---------------------------------------------------------------------------------------------------
BENCH_NAMES = ["Empty", "Ary1", "Ary16", "Ary256", "Ary512", "Ary1024", "Ary4096", "RunFull", "RunSplit", "Run16", "Run16Small",
               "Run256", "Run256Small", "Run1024", "BM512", "BM1024", "BM4096", "BM4097", "BM32768", "BM65000"]


def bench_archetype(rng, name):
    """-> (oracle Container in the named encoding, sorted value array)"""
    if name == "Empty":
        return O.Container.array(np.zeros(0, dtype=np.int64)), np.zeros(0, dtype=np.int64)
    if name.startswith("Ary"):
        v = np.sort(rng.choice(W, int(name[3:]), replace=False))
        return O.Container.array(v), v
    if name.startswith("BM"):
        v = np.sort(rng.choice(W, int(name[2:]), replace=False))
        w = np.zeros(1024, dtype=np.uint64)
        np.bitwise_or.at(w, v >> 6, np.uint64(1) << (v & 63).astype(np.uint64))
        return O.Container.bitmap(w), v
    if name == "RunFull":
        runs = [(0, W - 1)]
    elif name == "RunSplit":
        runs = [(0, 32700 + int(rng.integers(30))), (32768 + int(rng.integers(30)), W - 1)]
    else:
        small = name.endswith("Small")
        count = int(name[3:-5] if small else name[3:])
        stride = 65535 // (count + 1)
        lower, upper = (3, 3 + stride // 20) if small else (stride // 10, stride - 10)
        variance = upper - lower
        runs, nxt, prev = [], 0, 0
        for i in range(count):
            nxt += stride
            middle = (prev + nxt) // 2
            size = int(rng.integers(variance)) + lower
            start = middle + int(rng.integers(variance)) - size // 2
            last = start + size
            prev = nxt
            if runs and start <= runs[-1][1]:
                start = runs[-1][1] + 2
                last = max(last, start)
            runs.append((start, last))
    r = np.asarray(runs, dtype=np.int64)
    v = np.concatenate([np.arange(s, l + 1) for s, l in runs])
    return O.Container.run(r), v
