#!/usr/bin/env python3
"""Host-side model of the shared-memory cost of the 32-pattern content automaton (no GPU needed).

Replays what a warp of k_body does -- 32 records of one length-sorted group walked in lock step, one table lookup per byte and
lane -- on the synthetic corpus and the BASELINE configs[2] pattern batch, and counts, per warp-wide lookup, the conflict degree of
the 32 addresses (max number of distinct 4-byte words that fall into one of the 32 banks = shared-memory wavefronts) for a number
of table layouts.  Also prints the state-occupancy histogram and how compressible the transition table is.  The measured figure
of the shipped layout (ncu: 3.26-3.4 wavefronts per lookup) is reproduced by the first line.  The last section replays a
per-lane early exit for k_body (a lane stops once its content verdicts are decided) over the groups of one window; DESIGN
5.1 gives what it measured on the GPU.

    python tools/sim_lookup.py [groups]
"""
import os
import re
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench                                                    # noqa: E402
from fei_b200 import synth                                      # noqa: E402
from fei_b200.regexc import Pattern, compile_patterns          # noqa: E402


def main():
    groups = int(sys.argv[1]) if len(sys.argv) > 1 else 24
    d = compile_patterns([Pattern("regex", p, re.IGNORECASE) for p in bench.BATCH32])
    T, C, cls = d.trans, d.ctrans, d.cls
    n, nc = C.shape
    print(f"automaton: {n} states, {nc} byte classes ({int((cls < 29).sum())} ASCII bytes in {len(set(cls[:128].tolist()))} classes), "
          f"{int((d.out != 0).sum())} accepting states, {len(set(d.out[d.out != 0].tolist()))} distinct output masks")
    recs = [synth.record(bench.SEED, i)["body"] for i in range(4096)]
    lens = np.array([len(b) for b in recs])
    order = np.argsort(-((lens + 15) // 16), kind="stable")                      # one 4096-record window, sorted like the tiler sorts it
    # ---- state occupancy
    occ = np.zeros(n, dtype=np.int64)
    total = 0
    for r in recs[:512]:
        s = d.start
        for b in np.frombuffer(r, dtype=np.uint8):
            s = T[s, b]; occ[s] += 1
        total += len(r)
    cum = np.cumsum(np.sort(occ)[::-1]) / total
    print("state occupancy (share of byte steps spent in the k most visited states): " + ", ".join(f"top {k}: {cum[k - 1]:.2f}" for k in (1, 8, 32, 64, 96, 128, 256)))
    print(f"start state {occ[d.start] / total:.3f}; an accepting state is entered on {occ[d.out != 0].sum() / total:.3f} of the byte steps "
          f"(so on {1 - (1 - occ[d.out != 0].sum() / total) ** 32:.2f} of the warp steps some lane records a match)")
    root = C[d.start]
    print(f"entries that differ from the start state's row: {(C != root[None, :]).sum()} of {C.size} ({(C != root[None, :]).sum() / n:.1f} per state)")
    inc = {}
    for s in range(n):
        for c in range(nc):
            inc.setdefault(int(C[s, c]), set()).add(c)
    exp2 = 0
    for p in range(nc):
        members = [t for t, v in inc.items() if p in v and len(v) == 1]
        if members:
            sub = C[members]
            for c in range(nc):
                _v, cnt = np.unique(sub[:, c], return_counts=True)
                exp2 += len(members) - cnt.max()
    print(f"entries that differ from 'the row shared by all states entered on the same byte class': {exp2} ({exp2 / n:.2f} per state: the automaton is "
          f"'the pattern's next character, else a function of the last two characters')")
    # ---- lock-step traces
    traces = []
    for g in range(groups):
        lo = (g * 160) % (4096 - 32)
        ids = order[lo:lo + 32]
        L = min(min(len(recs[i]) for i in ids), 1500)
        B = np.stack([np.frombuffer(recs[i][:L], dtype=np.uint8) for i in ids], 1).astype(np.int64)
        S = np.zeros((L, 32), dtype=np.int64)
        s = np.full(32, d.start)
        for t in range(L):
            S[t] = s
            s = T[s, B[t]]
        traces.append((S, B))

    def degree(word_addr):
        deg = np.zeros(word_addr.shape[0], dtype=np.int64)
        for t in range(word_addr.shape[0]):
            deg[t] = np.bincount(np.unique(word_addr[t]) % 32, minlength=32).max()
        return deg

    def report(name, fn):
        degs = np.concatenate([degree(fn(S, B)) for S, B in traces])
        print(f"  {name:64s} {degs.mean():.2f} wavefronts per lookup")

    tile_perm = lambda b: b ^ ((b >> 1) & 0x20)
    c32 = np.where(cls < 29, cls, 0)                                              # ASCII fast path: 29 classes in 32 columns
    print("conflict degree per warp-wide lookup (one table lookup per byte and lane):")
    report("shipped: byte-indexed u16 rows, 129 words apart (178 KB)", lambda S, B: S * 129 + tile_perm(B) // 2)
    report("class-indexed u16 rows (47 classes)", lambda S, B: S * 25 + cls[B] // 2)
    report("class-indexed u16, 32 columns (22 KB)", lambda S, B: S * 17 + c32[B] // 2)
    report("class-indexed u8, 32 columns (11 KB)", lambda S, B: S * 9 + c32[B] // 4)

    def copies(k, stride_words, per_word):
        bw = 32 // k                                                              # copy c = lane % k lives in banks [c * bw, (c + 1) * bw)
        def fn(S, B):
            w = S * stride_words + c32[B] // per_word
            c = np.arange(32)[None, :] % k
            return (w // bw) * 32 + c * bw + (w % bw)
        return fn
    for k in (2, 4, 8, 16, 32):
        report(f"u16 x 32 columns, {k} copies, each confined to {32 // k} banks ({22 * k} KB)", copies(k, 17, 2))
    for k in (8, 16, 32):
        report(f"u8 x 32 columns, {k} copies, each confined to {32 // k} banks ({11 * k} KB)", copies(k, 9, 4))
    print("a byte -> class lookup (256-byte table, or one private copy per lane) costs one more wavefront per byte on top of the class-indexed rows")

    # ---- bank-private replicas of the HOT rows only (lane l keeps its copy of the K most visited states' rows in bank l), every other
    # state in the shared class-indexed table: hot lanes never collide with each other, but cold lanes land on any bank
    hot_rank = np.full(n, -1, dtype=np.int64)
    by_occ = np.argsort(-occ, kind="stable")
    for K in (32, 64, 128):
        hot_rank[:] = -1
        hot_rank[by_occ[:K]] = np.arange(K)
        one = []; two = []; share = []
        for S, B in traces:
            hot = hot_rank[S] >= 0
            shared_word = S * 17 + c32[B] // 2
            lanes = np.arange(32)
            for t in range(S.shape[0]):
                h = hot[t]
                load = np.zeros(32, dtype=np.int64)
                load[lanes[h]] += 1                                                # one private word per hot lane, in its own bank
                cold_words = np.unique(shared_word[t][~h])
                cold_load = np.bincount(cold_words % 32, minlength=32)
                one.append((load + cold_load).max())
                two.append((1 if h.any() else 0) + (cold_load.max() if len(cold_words) else 0))
            share.append(hot.mean())
        print(f"  top-{K} rows private per lane ({K * 32 * 2 * 32 // 1024} KB) + shared class-indexed table: {np.mean(share):.2f} of the lanes hot; "
              f"one mixed LDS {np.mean(one):.2f} wavefronts, hot and cold as two LDS {np.mean(two):.2f} (plus the byte -> class lookup)")

    # ---- splitting the pattern set (one read of the bytes feeds k sub-automata, each with its own table and its own lookup per byte)
    for k in (2, 4):
        parts = [bench.BATCH32[i::k] for i in range(k)]
        subs = [compile_patterns([Pattern("regex", p, re.IGNORECASE) for p in part]) for part in parts]
        states = [x.ctrans.shape[0] for x in subs]
        u8 = all(n_ <= 256 for n_ in states)
        kb = sum(n_ * 32 * (1 if u8 else 2) for n_ in states) / 1024
        copies = int(227 // kb) if kb else 0
        per = 1.0 if copies >= 32 else 2.0 if copies >= 16 else 2.9 if copies >= 8 else 3.2
        print(f"  {k} sub-automata of {32 // k} patterns: {states} states, class-indexed {'u8' if u8 else 'u16'} tables {kb:.1f} KB together -> at most {copies} bank-confined copies "
              f"(~{per:.1f} wavefronts per lookup), but {k} lookups per byte = ~{k * per:.1f} wavefronts per byte (plus the byte -> class lookup)")

    early_exit_model(d, recs, order, tile_perm)


def early_exit_model(d, recs, order, tile_perm):
    """A per-lane early exit for k_body, replayed on the 128 groups of window 0: a lane stops at the end of the 16-byte row in which the
    out[] masks of the states it has visited cover every content bit its queries read (all 32 here).  Counts, with and
    without the exit, the record bytes stepped through the automaton, the warp steps (16 per row in which some lane is
    still stepping) and the LDS wavefronts of the shipped layout, counting only the lanes that step."""
    need = (1 << d.n_patterns) - 1
    lanes = np.arange(32)
    tot = {"bytes": [0, 0], "steps": [0, 0], "wavefronts": [0, 0], "lookups": [0, 0]}
    early = n_rec = 0
    for g in range(len(order) // 32):
        ids = order[32 * g:32 * g + 32]
        lens = np.array([len(recs[i]) for i in ids])
        L = int(lens.max())
        B = np.zeros((L, 32), dtype=np.int64)
        for j, i in enumerate(ids):
            B[:lens[j], j] = np.frombuffer(recs[i], dtype=np.uint8)
        S = np.zeros((L, 32), dtype=np.int64)                        # state before byte t
        s = np.full(32, d.start)
        acc = np.full(32, int(d.out[d.start]), dtype=np.int64)
        done_at = np.full(32, -1)                                    # first byte after which acc covers need
        for t in range(L):
            S[t] = s
            s = d.trans[s, B[t]]
            acc |= d.out[s].astype(np.int64)
            newly = (done_at < 0) & ((acc & need) == need) & (t < lens)
            done_at[newly] = t
        rows = (lens + 15) // 16
        stop_rows = np.where(done_at >= 0, done_at // 16 + 1, rows)  # rows a lane runs with the exit
        n_rec += 32
        early += int((stop_rows < rows).sum())
        word = S * 129 + tile_perm(B) // 2
        t = np.arange(L)[:, None]
        for k, lane_rows in enumerate((rows, stop_rows)):
            active = (t < lens[None, :]) & (t < 16 * lane_rows[None, :])
            tot["bytes"][k] += int(active.sum())
            tot["steps"][k] += 16 * int(lane_rows.max())
            w = np.where(active, word, -1 - lanes[None, :])          # inactive lanes: distinct negative words, no bank
            srt = np.sort(w, axis=1)
            first = np.ones_like(srt, dtype=bool)
            first[:, 1:] = srt[:, 1:] != srt[:, :-1]
            first &= srt >= 0
            cnt = np.zeros((L, 32), dtype=np.int64)
            r_idx, c_idx = np.nonzero(first)
            np.add.at(cnt, (r_idx, srt[r_idx, c_idx] % 32), 1)
            deg = cnt.max(axis=1)
            tot["wavefronts"][k] += int(deg.sum())
            tot["lookups"][k] += int((deg > 0).sum())
    ratio = {k: v[1] / v[0] for k, v in tot.items()}
    print(f"per-lane early exit model (all {d.n_patterns} content bits needed; window 0, {len(order) // 32} groups in tiler order):")
    print(f"  records decided before their last row: {early / n_rec:.3f}")
    print(f"  lane-bytes through the automaton: {ratio['bytes']:.3f} of the full scan")
    print(f"  LDS wavefronts (active lanes only, byte-indexed u16 rows 129 words apart): {ratio['wavefronts']:.3f} of the full scan "
          f"({tot['wavefronts'][0] / tot['lookups'][0]:.2f} -> {tot['wavefronts'][1] / tot['lookups'][1]:.2f} per warp-wide lookup)")
    print(f"  warp steps: {ratio['steps']:.3f} of the full scan")


if __name__ == "__main__":
    main()
