"""CPU model of a serialized content automaton (fei_b200/program.py serialize_dfa, include/feiscan_prog.h fei_prog_dfa):
reads the descriptor and tables out of a program blob and steps a body the way the scan kernels do, so a test can tell
a wrong table from a wrong kernel."""
import struct

import numpy as np

from fei_b200.program import tile_byte_perm

_TILE_BYTE = tile_byte_perm(np.arange(256)).tolist()


class BlobDfa:
    def __init__(self, blob: bytes, off: int):
        (self.n_states, self.n_cols, self.start, self.n_acc, off_trans, _trans_bytes, off_out, off_endout, off_cls,
         self.n_patterns, self.empty_acc, self.table_bytes, self.row_stride, self.sticky) = struct.unpack_from("<14I", blob, off)
        trans = np.frombuffer(blob, np.uint16, self.n_states * self.row_stride, off_trans).reshape(self.n_states, self.row_stride)
        self.trans = trans.tolist()
        self.out = np.frombuffer(blob, np.uint32, self.n_states, off_out).tolist()
        self.endout = np.frombuffer(blob, np.uint32, self.n_states, off_endout).tolist()
        self.cls = np.frombuffer(blob, np.uint8, 256, off_cls).tolist()
        self.direct = self.n_cols == 256

    @classmethod
    def from_program(cls, prog: bytes) -> "BlobDfa":
        return cls(prog, struct.unpack_from("<I", prog, 40)[0])          # fei_prog_hdr.off_body_dfa

    def run(self, body: bytes) -> int:
        """Content bits of `body` (the text as stored: the kernels read tile bytes, i.e. tile_byte_perm of each byte)."""
        s = self.start
        acc = self.out[s] if s < self.n_acc else 0
        absorbing = self.sticky - 1 if self.sticky not in (0, 0xFFFFFFFF) else -1
        for b in body:
            if s == absorbing:                                               # a sticky scan stops at its matched state
                break
            c = _TILE_BYTE[b]
            s = self.trans[s][c if self.direct else self.cls[c]]
            if s < self.n_acc:
                acc |= self.out[s]
        return acc | self.endout[s]
