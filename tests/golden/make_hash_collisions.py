"""Regenerates hash_collisions.json: pairs of distinct 8-byte ASCII cells that the text group-by
(``k_hash_count_str``, learningorchestra_b200/csrc/kernels.cuh) cannot tell apart by their slot tag.

A slot of the text hash table holds the top 33 bits of the cell's 64-bit hash (``hash_bytes``) and the row of the
group's representative; a probe whose tag matches compares the bytes.  Each pair here has the same 33-bit tag AND the
same start slot, ``splitmix64(hash) & (slots - 1)``, in a ``TABLE_SLOTS``-slot table (the size of the table of every
column of at most 512 cells), while the full 64-bit hashes differ.  So both cells of a pair probe the same slot and
only the byte comparison keeps them in separate groups.

The search runs a numpy port of ``hash_bytes`` over ``2 ** SEARCH_BITS`` distinct strings of 8 letters 'a'..'p' (one
per nibble of a bijective scramble of the index); it takes a few seconds.  tests/test_groupby_prepass_cpu.py checks every pair
against the real ``hash_bytes`` compiled from kernels.cuh, so a wrong port cannot pass unnoticed.

    python tests/golden/make_hash_collisions.py
"""
import json
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
OUT = HERE / "hash_collisions.json"
TABLE_SLOTS = 1024
LENGTH = 8
SEARCH_BITS = 23
TAG_SHIFT = 31                       # tag = hash >> 31: the top 33 bits

FNV_OFFSET = np.uint64(0xCBF29CE484222325)
FNV_PRIME = np.uint64(0x100000001B3)


def splitmix64(z):
    z = np.asarray(z, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = z + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def hash_bytes(cells: np.ndarray) -> np.ndarray:
    """cells: uint8 [n, length] -> the 64-bit hash of each row (FNV-1a seeded with the length, then splitmix64)."""
    n, length = cells.shape
    h = np.full(n, FNV_OFFSET ^ np.uint64(length), dtype=np.uint64)
    with np.errstate(over="ignore"):
        for i in range(length):
            h = (h ^ cells[:, i].astype(np.uint64)) * FNV_PRIME
    return splitmix64(h)


def candidates(bits: int) -> np.ndarray:
    """2**bits distinct strings: the 8 nibbles of (index * odd constant) mod 2^32, each as a letter 'a'..'p'."""
    x = (np.arange(1 << bits, dtype=np.uint64) * np.uint64(0x9E3779B1)) & np.uint64(0xFFFFFFFF)
    nib = np.stack([(x >> np.uint64(28 - 4 * i)) & np.uint64(0xF) for i in range(LENGTH)], axis=1)
    return (nib + ord("a")).astype(np.uint8)


def search(bits: int = SEARCH_BITS):
    cells = candidates(bits)
    h = hash_bytes(cells)
    tag = h >> np.uint64(TAG_SHIFT)
    order = np.argsort(tag, kind="stable")
    st = tag[order]
    same = np.flatnonzero(st[1:] == st[:-1])
    pairs = []
    for i in same:
        a, b = int(order[i]), int(order[i + 1])
        if h[a] == h[b]:
            continue
        sa = int(splitmix64(h[a]) & np.uint64(TABLE_SLOTS - 1))
        sb = int(splitmix64(h[b]) & np.uint64(TABLE_SLOTS - 1))
        if sa == sb:
            pairs.append({"a": cells[a].tobytes().decode("ascii"), "b": cells[b].tobytes().decode("ascii"),
                          "hash_a": f"{int(h[a]):016x}", "hash_b": f"{int(h[b]):016x}",
                          "tag": f"{int(tag[a]):09x}", "slot": sa})
    return sorted(pairs, key=lambda p: p["a"])


def main():
    pairs = search()
    OUT.write_text(json.dumps({"table_slots": TABLE_SLOTS, "length": LENGTH, "tag_shift": TAG_SHIFT, "pairs": pairs},
                              indent=1) + "\n")
    print(f"{len(pairs)} pairs -> {OUT}")


if __name__ == "__main__":
    main()
