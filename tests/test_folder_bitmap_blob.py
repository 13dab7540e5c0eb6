"""Folder sets as a program carries them (CPU suite): a set that holds a folder id of 64 or above is a uint32 bitmap in the
program head at fei_prog_cond.off_set_words (include/feiscan_prog.h); a set of ids below 64 is set64 alone and the program is
byte-identical to one written without bitmap support.  A model of the head kernels' test, run over the blob, must agree with
the set for every folder id."""
import struct

import pytest

from fei_b200.program import C_FOLDER_SET, C_SLOT, C_STATUS_SET, Cond, ProgramBuilder
from fei_b200.regexc import Pattern

_HDR = struct.Struct("<24I")
_COND = struct.Struct("<6B2xqQ2I")


def _conds(blob):
    h = _HDR.unpack_from(blob, 0)
    n_conds, off_conds, head_bytes = h[4], h[5], h[19]
    return [_COND.unpack_from(blob, off_conds + 32 * k) for k in range(n_conds)], head_bytes, h


def _in_set(blob, cond, fid):
    """What eval_meta_cond<kFolderBits = true> reads for a FEI_C_FOLDER_SET condition."""
    set64, off, n_words = cond[7], cond[8], cond[9]
    if not off:
        return fid < 64 and bool(set64 >> fid & 1)
    if fid >= 32 * n_words:
        return False
    return bool(struct.unpack_from("<I", blob, off + 4 * (fid >> 5))[0] >> (fid & 31) & 1)


@pytest.mark.parametrize("ids", [[0, 5, 63], [64], [1, 63, 64, 65, 100, 127, 128, 500], [700], list(range(0, 300, 7))])
def test_folder_set_bitmap_layout(ids):
    bits = sum(1 << i for i in ids)
    pb = ProgramBuilder()
    pb.add_query([Cond(C_FOLDER_SET, set64=bits)])
    pb.add_query([Cond(C_STATUS_SET, set64=0b101), Cond(C_FOLDER_SET, set64=bits | 1 << 3)])
    pb.add_query([Cond(C_SLOT, pattern=Pattern("contains", "x"), field="Subject"), Cond(C_FOLDER_SET, set64=1 << 2)])
    blob = pb.build()
    conds, head_bytes, h = _conds(blob)
    folder_sets = [(c, want) for c, want in zip(conds, [bits, 0b101, bits | 1 << 3, 0, 1 << 2]) if c[0] == C_FOLDER_SET]
    assert len(folder_sets) == 3
    taken = []
    for c, want in folder_sets:
        off, n_words = c[8], c[9]
        assert c[7] == want & (1 << 64) - 1                    # set64 keeps ids 0..63 either way
        if want >> 64:
            assert off % 16 == 0 and off + 4 * n_words <= head_bytes and off >= h[6] + 16 * h[3]      # after the query table
            assert n_words == (want.bit_length() + 31) // 32
            taken.append((off, off + 4 * n_words))
        else:
            assert (off, n_words) == (0, 0)
        for fid in range(0, 1100):
            assert _in_set(blob, c, fid) == bool(want >> fid & 1), (ids, fid)
    # bitmaps overlap neither each other nor any section the header points at
    taken.sort()
    assert all(a[1] <= b[0] for a, b in zip(taken, taken[1:]))
    sections = [h[k] for k in (5, 6, 8, 9, 10, 11, 12, 13, 14, 20, 21, 22, 23) if h[k]]
    assert not any(a <= s < b for s in sections for a, b in taken)
    status = next(c for c in conds if c[0] == C_STATUS_SET)
    assert status[7:] == (0b101, 0, 0)


def test_small_folder_sets_write_the_same_blob():
    """No bitmap below id 64: the condition's last eight bytes stay zero and nothing is appended to the head."""
    def prog(bits):
        pb = ProgramBuilder()
        pb.add_query([Cond(C_FOLDER_SET, set64=bits), Cond(C_SLOT, pattern=Pattern("contains", "a"), field="Tags")])
        return pb.build()
    small = prog((1 << 63) | 0b1011)
    conds, head_bytes, _h = _conds(small)
    assert conds[0][8:] == (0, 0)
    big = prog((1 << 64) | (1 << 63) | 0b1011)
    assert len(big) == len(small) + 16                          # one 16-byte padded bitmap of 3 words
    assert _conds(big)[1] == head_bytes + 16
