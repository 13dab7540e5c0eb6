"""CPU model of a serialized content position automaton (fei_b200/program.py serialize_nfa, include/feiscan_prog.h
fei_prog_nfa): reads the section out of a program blob and steps a stored body the way k_body_nfa does -- undo the tile byte
permutation, decode UTF-8, look the class up (ASCII table, else a binary search over the range table), step the W-word
vector -- next to the program's body DFA when it has one, so a test can tell a wrong table from a wrong kernel.  The content
section of a version-3 program also has counter positions (fei_prog_nfa_ctr right behind the descriptor), stepped the way
k_body_nfa's counted instances do -- per counter position P with bound k,
    entered = F[P];  D'[P] = B[class][P] && (entered || (D[P] && age_P < k));  age_P = entered ? 1 : age_P + 1"""
import struct

import numpy as np

from fei_b200.program import VERSION_CTR, tile_byte_perm
from tests.blob_model import BlobDfa

_TILE_BYTE = tile_byte_perm(np.arange(256)).tolist()


class BlobNfa:
    def __init__(self, blob: bytes, off: int, counters: bool = False):
        (self.W, self.n_pos, self.n_classes, self.n_ranges, self.n_follow, self.n_accept, self.n_patterns, self.first_bit,
         off_ascii, off_lo, off_rck, off_b, off_masks, off_follow, off_accept, self.table_bytes) = struct.unpack_from("<16I", blob, off)
        W = self.W
        u32 = lambda o, k: np.frombuffer(blob, np.uint32, k, o).tolist()           # noqa: E731

        def vec(ws):
            return sum(int(w) << (32 * k) for k, w in enumerate(ws))

        self.ascii = np.frombuffer(blob, np.uint16, 128, off_ascii).tolist()
        self.range_lo = u32(off_lo, self.n_ranges)
        self.range_ck = np.frombuffer(blob, np.uint16, self.n_ranges, off_rck).tolist()
        b = u32(off_b, self.n_classes * W)
        self.cls_b = [vec(b[c * W:(c + 1) * W]) for c in range(self.n_classes)]
        m = u32(off_masks, 3 * W)
        self.shift, self.self_loop, self.start = vec(m[:W]), vec(m[W:2 * W]), vec(m[2 * W:])
        f = u32(off_follow, self.n_follow * (2 * W + 1))
        self.follow = [(vec(r[:W]), vec(r[W:2 * W]), r[2 * W]) for r in (f[g * (2 * W + 1):(g + 1) * (2 * W + 1)] for g in range(self.n_follow))]
        a = u32(off_accept, self.n_accept * (W + 2))
        self.accept = [(vec(r[:W]), r[W], r[W + 1] & 0xFF, bool(r[W + 1] >> 8)) for r in (a[g * (W + 2):(g + 1) * (W + 2)] for g in range(self.n_accept))]
        self.counters = []                                                # (position, bound) of each counter position
        if counters:
            n, off_ctr = struct.unpack_from("<2I", blob, off + 64)                 # fei_prog_nfa_ctr
            tab = struct.unpack_from(f"<{2 * n}I", blob, off_ctr)
            self.counters = [(tab[2 * i], tab[2 * i + 1]) for i in range(n)]

    @classmethod
    def from_program(cls, prog: bytes) -> "BlobNfa":
        """The content section (fei_prog_hdr.off_body_nfa), with its counters when the program is version 3."""
        return cls(prog, struct.unpack_from("<I", prog, 88)[0], struct.unpack_from("<I", prog, 4)[0] == VERSION_CTR)

    def class_kind(self, cp: int) -> int:
        if cp < 0x80:
            return self.ascii[cp]
        lo, hi = 0, self.n_ranges - 1
        while lo < hi:
            mid = (lo + hi + 1) >> 1
            if self.range_lo[mid] <= cp:
                lo = mid
            else:
                hi = mid - 1
        return self.range_ck[lo]

    def _accepts(self, d: int, ctx: int, at_end: bool) -> int:
        acc = 0
        for src, m, bit, end_only in self.accept:
            if (at_end or not end_only) and m & ctx and d & src:
                acc |= 1 << bit
        return acc

    def run(self, body: bytes) -> int:
        """Content bits (first_bit ...) of a body given as its text: each byte goes through the tile permutation and back,
        as the kernel reads it."""
        d, prev, acc = self.start, 0, 0
        cp, need = 0, 0
        age = [0] * len(self.counters)
        for raw in body:
            byte = _TILE_BYTE[_TILE_BYTE[raw]]
            if byte < 0x80:
                cp, need = byte, 0
            elif byte >= 0xC0:
                need = 3 if byte >= 0xF0 else 2 if byte >= 0xE0 else 1
                cp = byte & (0x3F >> need)
                continue
            else:
                cp = (cp << 6) | (byte & 0x3F)
                need -= 1
                if need:
                    continue
            ck = self.class_kind(cp)
            c, kind = ck & 0xFF, ck >> 8
            ctx = 1 << (prev * 5 + kind)
            acc |= self._accepts(d, ctx, False)
            nd = ((d << 1) & self.shift) | (d & self.self_loop)
            for src, dst, m in self.follow:
                if m & ctx and d & src:
                    nd |= dst
            keep = 0
            for i, (p, k) in enumerate(self.counters):
                if d >> p & 1 and age[i] < k:
                    keep |= 1 << p
                age[i] = 1 if nd >> p & 1 else age[i] + 1
            d = (nd | keep) & self.cls_b[c]
            prev = kind
        return acc | self._accepts(d, 1 << (prev * 5), True)


def program_content_bits(prog: bytes, body: bytes) -> int:
    """The content verdict k_body_nfa computes for `body`: the body DFA's bits (if any) | the position automaton's."""
    acc = BlobNfa.from_program(prog).run(body)
    if struct.unpack_from("<I", prog, 40)[0]:                            # fei_prog_hdr.off_body_dfa
        acc |= BlobDfa.from_program(prog).run(body)
    return acc
