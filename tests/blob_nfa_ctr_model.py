"""CPU model of a serialized content position automaton with counters (include/feiscan_prog.h fei_prog_nfa_ctr, version-3
programs): tests/blob_nfa_model.py's section reader plus the counter descriptor right behind the section, stepped the way
k_body_nfa's counted instances do -- per counter position P with bound k,
    entered = F[P];  D'[P] = B[class][P] && (entered || (D[P] && age_P < k));  age_P = entered ? 1 : age_P + 1"""
import struct

from tests.blob_model import BlobDfa
from tests.blob_nfa_model import _TILE_BYTE, BlobNfa


class BlobNfaCtr(BlobNfa):
    def __init__(self, blob: bytes, off: int, with_counters: bool):
        super().__init__(blob, off)
        self.counters = []
        if with_counters:
            n, off_ctr = struct.unpack_from("<2I", blob, off + 64)                 # fei_prog_nfa_ctr
            tab = struct.unpack_from(f"<{2 * n}I", blob, off_ctr)
            self.counters = [(tab[2 * i], tab[2 * i + 1]) for i in range(n)]

    @classmethod
    def from_program(cls, prog: bytes) -> "BlobNfaCtr":
        version, = struct.unpack_from("<I", prog, 4)
        return cls(prog, struct.unpack_from("<I", prog, 88)[0], version == 3)

    def run(self, body: bytes) -> int:
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
    acc = BlobNfaCtr.from_program(prog).run(body)
    if struct.unpack_from("<I", prog, 40)[0]:                            # fei_prog_hdr.off_body_dfa
        acc |= BlobDfa.from_program(prog).run(body)
    return acc
