#!/usr/bin/env python
"""Census of the headline workload (realdata all-pairs): work items of k_compute_items by kind,
type pair and size class, per dataset — what the kernel's time has to be spent on — and the
pass-through containers of each op (keys in one operand only: OR / XOR keep both sides', ANDNOT
the left side's) with their stored bytes, 16-byte rounded as in the slab.  Non-lazy batch ops
share these with their operands instead of copying them."""
import collections
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import croaring_b200.datasets as dsm  # noqa: E402


def index(blob):
    cookie = int(np.frombuffer(blob[:4], dtype="<u4")[0])
    if (cookie & 0xFFFF) == 12347:
        n = (cookie >> 16) + 1
        nb = (n + 7) // 8
        isrun = np.unpackbits(np.frombuffer(blob[4:4 + nb], dtype=np.uint8), bitorder="little")[:n].astype(bool)
        pos = 4 + nb
        hasrun = True
    else:
        n = int(np.frombuffer(blob[4:8], dtype="<u4")[0])
        isrun = np.zeros(n, dtype=bool)
        pos = 8
        hasrun = False
    kc = np.frombuffer(blob[pos:pos + 4 * n], dtype="<u2").reshape(n, 2)
    pos += 4 * n
    if (not hasrun) or n >= 4:
        pos += 4 * n
    keys = kc[:, 0].astype(np.int64)
    cards = kc[:, 1].astype(np.int64) + 1
    types = np.where(isrun, 3, np.where(cards > 4096, 1, 2))
    lens = np.zeros(n, dtype=np.int64)
    p = pos
    for i in range(n):
        if isrun[i]:
            nr = int(np.frombuffer(blob[p:p + 2], dtype="<u2")[0])
            lens[i] = nr
            p += 2 + 4 * nr
        elif cards[i] > 4096:
            lens[i] = 1024
            p += 8192
        else:
            lens[i] = cards[i]
            p += 2 * cards[i]
    return keys, types, cards, lens


def stored16(types, cards, lens):
    """slab bytes of each container: bitset 8192, array 2 x card, run 4 x runs, rounded up to 16"""
    b = np.where(types == 1, 8192, np.where(types == 2, 2 * cards, 4 * lens))
    return (b + 15) // 16 * 16


def main():
    T = {1: "B", 2: "A", 3: "R"}
    for ds in ["census1881", "weather_sept_85", "wikileaks-noquotes"]:
        blobs = dsm.load_realdata(ds)
        ix = [index(b) for b in blobs]
        nct = collections.Counter()
        for k, t, c, l in ix:
            for tt in t:
                nct[T[int(tt)]] += 1
        print(f"== {ds}: containers by type {dict(nct)}; per bitmap {np.mean([len(k) for k, *_ in ix]):.1f}")
        arr_cards = np.concatenate([c[t == 2] for k, t, c, l in ix]) if nct["A"] else np.zeros(0)
        run_lens = np.concatenate([l[t == 3] for k, t, c, l in ix]) if nct["R"] else np.zeros(0)
        if len(arr_cards):
            print(f"   array cards: mean {arr_cards.mean():.0f} median {np.median(arr_cards):.0f} p90 {np.percentile(arr_cards, 90):.0f}")
        if len(run_lens):
            print(f"   run lens: mean {run_lens.mean():.1f} median {np.median(run_lens):.0f} p90 {np.percentile(run_lens, 90):.0f} max {run_lens.max()}")
        cells = collections.Counter()
        sizes = collections.defaultdict(list)
        copies = collections.Counter()
        sb = [stored16(t, c, l) for k, t, c, l in ix]
        pt_n = {"left": 0, "right": 0}
        pt_b = {"left": 0, "right": 0}
        n = len(ix)
        for i in range(n):
            ki, ti, ci, li = ix[i]
            for j in range(i + 1, n):
                kj, tj, cj, lj = ix[j]
                _, ai, aj = np.intersect1d(ki, kj, assume_unique=True, return_indices=True)
                for a, b in zip(ai, aj):
                    tp = T[int(ti[a])] + T[int(tj[b])]
                    cells[tp] += 1
                    if len(sizes[tp]) < 20000:
                        sizes[tp].append((int(ci[a]), int(cj[b]), int(li[a]), int(lj[b])))
                # pass-through (or / xor): unmatched on both sides
                mi = np.ones(len(ki), bool)
                mi[ai] = False
                mj = np.ones(len(kj), bool)
                mj[aj] = False
                for t in ti[mi]:
                    copies[T[int(t)]] += 1
                for t in tj[mj]:
                    copies[T[int(t)]] += 1
                pt_n["left"] += int(mi.sum())
                pt_n["right"] += int(mj.sum())
                pt_b["left"] += int(sb[i][mi].sum())
                pt_b["right"] += int(sb[j][mj].sum())
        tot = sum(cells.values())
        print(f"   matched cells {tot} ({tot / 19900:.1f}/pair), pass-through {sum(copies.values())} ({sum(copies.values()) / 19900:.1f}/pair) {dict(copies)}")
        for op, sides in (("or / xor", ("left", "right")), ("andnot", ("left",))):
            cnt_op = sum(pt_n[x] for x in sides)
            b_op = sum(pt_b[x] for x in sides)
            print(f"   pass-through per {op} call: {cnt_op} containers, {b_op} stored bytes ({b_op / 1e9:.3f} GB); "
                  f"a copy reads and writes them: {2 * b_op / 1e9:.3f} GB")
        for tp, cnt in cells.most_common():
            s = np.array(sizes[tp])
            print(f"     {tp}: {cnt:8d} ({100 * cnt / tot:5.1f}%)  cardA mean {s[:, 0].mean():7.0f} cardB mean {s[:, 1].mean():7.0f} "
                  f"lenA {s[:, 2].mean():6.0f} lenB {s[:, 3].mean():6.0f}  sum<=2032: {100 * np.mean(s[:, 0] + s[:, 1] <= 2032):.0f}% sum<=4096: {100 * np.mean(s[:, 0] + s[:, 1] <= 4096):.0f}%")


if __name__ == "__main__":
    main()
