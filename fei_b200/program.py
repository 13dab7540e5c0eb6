"""Predicate programs: queries -> the binary blob `fei_scan_*` takes (include/feiscan_prog.h).

A program holds up to 32 queries; a query is the AND of conditions.  Every string-valued
condition becomes one output bit of the multi-output byte DFA of the field it reads
(fei_b200.regexc), so all conditions of all queries on one field cost one pass over it.
"""
from __future__ import annotations

import struct
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from .regexc import Dfa, Pattern, PatternTooLarge, Pna, compile_patterns, compile_positions, compile_positions_counted

MAGIC, VERSION, VERSION_NFA, VERSION_CTR = 0x50494546, 1, 2, 3
C_CONST, C_BODY, C_SLOT, C_FLAGS, C_NAME, C_DATE_CMP, C_FOLDER_SET, C_STATUS_SET, C_RECBITS, C_TS_CMP = range(10)
CMP = {">": 0, "<": 1, ">=": 2, "<=": 3, "=": 4, "!=": 5}
NAME_FILENAME, NAME_ID, NAME_HOST, NAME_TS_STR, NAME_DATE_STR = 0, 1, 2, 3, 4     # 3 / 4: str(metadata["timestamp"]) / str(metadata["date"]), formatted by the kernels
MAX_AUX = 4                            # aux verdict columns per corpus (FEI_C_RECBITS)
SMEM_TABLE_LIMIT = 200 * 1024          # body automaton must fit the CTA's shared memory
BODY_SMEM_LIMIT = 220 * 1024           # scan.cu: dynamic shared memory of a body kernel (content DFA + position automaton tables)
HEAD_SMEM_WINDOW = 32 * 1024           # scan.cu kHeadProgSmem: the program head the head kernels stage per CTA
HEAD_DIRECT_LIMIT = 12 * 1024          # a head automaton up to this size is stored byte-indexed


@dataclass(frozen=True)
class Cond:
    """One condition.  kind + what it reads:
       const(value) | body(pattern) | slot(field, mode, empty_if_missing, pattern) | flags(pattern)
       | name(which, pattern) | date_cmp(op, micros) | folder_set(bits) | status_set(bits)
       | recbits(which = aux column, negate) | ts_cmp(op, i64)"""
    kind: int
    pattern: Optional[Pattern] = None
    negate: bool = False
    field: str = ""              # header field name (slot)
    mode: int = 0                # slot: 0 = case-insensitive first key, 1 = exact key, 2 = any key (OR over all header values)
    empty_if_missing: bool = False
    if_missing: int = 0          # slot: 0/1 result when absent, 2 = next condition is the fallback
    which: int = 0               # name field
    op: int = 0                  # date_cmp
    i64: int = 0
    set64: int = 0               # folder / status set: bit k = id k (a folder set may hold ids of 64 and above)
    value: bool = False          # const


def const(v: bool) -> Cond:
    return Cond(C_CONST, value=bool(v))


def _pad16(b: bytearray) -> None:
    while len(b) % 16:
        b.append(0)


_DFA_CACHE: Dict[Tuple, Dfa] = {}
_DFA_FAIL: Dict[Tuple, str] = {}       # same keys: pattern sets whose DFA was refused (PatternTooLarge), with the reason
_PNA_CACHE: Dict[Tuple, Pna] = {}


def _remember(cache: Dict, key, value) -> None:
    if len(cache) >= 256:
        cache.pop(next(iter(cache)))
    cache[key] = value


def _pkey(p: Pattern) -> Tuple:
    return (p.kind, p.text, int(p.flags))


def cached_dfa(patterns: Sequence[Pattern], sticky: bool = False) -> Dfa:
    """compile_patterns, cached per process; a refusal (PatternTooLarge) is cached too, so a repeated query does not pay for
    the failed subset construction again (seconds for a bounded gap such as `.{0,60}`)."""
    sticky = sticky and len(patterns) == 1
    key = (tuple(_pkey(p) for p in patterns), sticky)
    d = _DFA_CACHE.get(key)
    if d is not None:
        return d
    why = _DFA_FAIL.get(key)
    if why is not None:
        raise PatternTooLarge(why)
    try:
        d = compile_patterns(patterns, sticky=sticky)
    except PatternTooLarge as e:
        _remember(_DFA_FAIL, key, str(e))
        raise
    _remember(_DFA_CACHE, key, d)
    return d


def cached_positions(patterns: Sequence[Pattern], counters: bool = False) -> Pna:
    """The position automaton of `patterns`, cached per process.  With `counters` (content), compile_positions_counted where
    the plain automaton is refused (long bounded gaps such as `a.{0,1000}b`); head fields keep the plain one."""
    key = (tuple(_pkey(p) for p in patterns), counters)
    a = _PNA_CACHE.get(key)
    if a is None:
        try:
            a = compile_positions(patterns)
        except PatternTooLarge:
            if not counters:
                raise
            a = compile_positions_counted(patterns)
        _remember(_PNA_CACHE, key, a)
    return a


def content_automaton(p: Pattern):
    """The automaton one pattern runs on the host: its DFA, or its position automaton when the DFA is refused.  Both have
    .run(bytes) -> mask: the empty-string verdict of a content condition without with_content, and the folder / status names
    search judges on the host."""
    try:
        return cached_dfa([p])
    except PatternTooLarge:
        return cached_positions([p], counters=True)


class _FieldDfa:
    """Patterns that read the same field, deduplicated -> output bits."""

    def __init__(self, what: str):
        self.what = what
        self.patterns: List[Pattern] = []
        self.index: Dict[Tuple, int] = {}

    def bit(self, p: Pattern) -> int:
        key = (p.kind, p.text, int(p.flags))
        b = self.index.get(key)
        if b is None:
            b = len(self.patterns)
            if b >= 32:
                raise NotImplementedError(f"more than 32 distinct patterns on {self.what} in one program")
            self.index[key] = b
            self.patterns.append(p)
        return b

    def compile(self, sticky: bool = False) -> Dfa:
        """Compiled automata are cached per process: repeated queries / the default filters skip the (host-side,
        Python) subset construction, which costs 10-900 ms for Unicode-class-heavy patterns."""
        return cached_dfa(self.patterns, sticky)


def tile_byte_perm(b: np.ndarray) -> np.ndarray:
    """Byte substitution applied to the body tiles at pack time (fei_b200/csrc/corpus.h): bit 5 ^= bit 6."""
    b = b.astype(np.int64)
    return b ^ ((b >> 1) & 0x20)


def serialize_dfa(d: Dfa, blob: bytearray, direct_limit: int = 0, tile_bytes: bool = False) -> int:
    """Append descriptor + tables; returns the descriptor offset.  States are renumbered so that
    states with a non-empty `out` come first (the kernels test `state < n_acc`, and the body kernel
    records accepting state k as bit k without a table lookup)."""
    n = d.n_states
    if n > 65535:
        raise NotImplementedError("automaton has more than 65535 states")
    accepting = d.out != 0
    order = np.concatenate([np.nonzero(accepting)[0], np.nonzero(~accepting)[0]])
    new_id = np.empty(n, dtype=np.int64)
    new_id[order] = np.arange(n)
    n_acc = int(accepting.sum())
    direct = direct_limit and n * 516 + n * 8 + 256 <= direct_limit
    cls = d.cls.astype(np.uint8)
    if direct:
        trans = new_id[d.trans[order]].astype(np.uint16)              # [n, 256]
        ncols = 256
        if tile_bytes:                                                # columns addressed by the stored (permuted) byte
            trans = trans[:, tile_byte_perm(np.arange(256))]
    else:
        trans = new_id[d.ctrans[order]].astype(np.uint16)             # [n, ncls]
        ncols = trans.shape[1]
        if tile_bytes:
            cls = cls[tile_byte_perm(np.arange(256))]
    # pad rows so that (row_stride / 2) is odd: state s starts at bank (s * stride/2) % 32, which walks
    # all 32 banks instead of piling every row onto the same ones (bank-conflict spreading)
    stride = ncols + (ncols & 1)
    if (stride // 2) % 2 == 0:
        stride += 2
    padded = np.zeros((n, stride), dtype=np.uint16)
    padded[:, :ncols] = trans
    trans = padded
    out = d.out[order].astype(np.uint32)
    endout = d.endout[order].astype(np.uint32)
    start = int(new_id[d.start])
    _pad16(blob)
    desc_off = len(blob)
    blob.extend(b"\0" * 64)
    _pad16(blob)
    off_trans = len(blob)
    blob.extend(trans.tobytes()); _pad16(blob)
    trans_bytes = len(blob) - off_trans
    off_out = len(blob); blob.extend(out.tobytes()); _pad16(blob)
    off_endout = len(blob); blob.extend(endout.tobytes()); _pad16(blob)
    off_cls = len(blob); blob.extend(cls.tobytes()); _pad16(blob)
    table_bytes = len(blob) - off_trans
    empty_acc = int(out[start]) | int(endout[start])
    sticky = 0
    if d.sticky_state >= -1:
        sticky = 0xFFFFFFFF if d.sticky_state < 0 else 1 + int(new_id[d.sticky_state])
    struct.pack_into("<16I", blob, desc_off, n, ncols, start, n_acc, off_trans, trans_bytes, off_out, off_endout,
                     off_cls, d.n_patterns, empty_acc, table_bytes, stride, sticky, 0, 0)
    return desc_off


def _table_bytes(d: Dfa, direct_limit: int) -> int:
    """fei_prog_dfa.table_bytes that serialize_dfa(d, blob, direct_limit) writes, without writing it."""
    n = d.n_states
    ncols = 256 if direct_limit and n * 516 + n * 8 + 256 <= direct_limit else d.ctrans.shape[1]
    stride = ncols + (ncols & 1)
    if (stride // 2) % 2 == 0:
        stride += 2
    return sum((x + 15) & ~15 for x in (2 * n * stride, 4 * n, 4 * n, 256))


def serialize_nfa(a: Pna, blob: bytearray, first_bit: int) -> int:
    """Append a fei_prog_nfa section (include/feiscan_prog.h); returns its offset.  Output bit k of the automaton becomes
    content bit first_bit + k.  An automaton with counters (content only) gets a fei_prog_nfa_ctr right behind the descriptor."""
    W = a.n_words
    if first_bit + a.n_patterns > 32:
        raise NotImplementedError("more than 32 content patterns in one program")

    def words(m: int) -> List[int]:
        return [(m >> (32 * k)) & 0xFFFFFFFF for k in range(W)]

    def table(arr: np.ndarray) -> int:
        off = len(blob)
        blob.extend(arr.tobytes()); _pad16(blob)
        return off

    _pad16(blob)
    desc_off = len(blob)
    blob.extend(b"\0" * (80 if a.counters else 64))                               # + fei_prog_nfa_ctr
    ck = lambda c: c | a.cls_kind[c] << 8                                          # noqa: E731
    off_ascii = table(np.array([ck(c) for c in a.ascii_cls], dtype=np.uint16))
    off_lo = table(np.array([lo for lo, _c in a.ranges], dtype=np.uint32))
    off_rck = table(np.array([ck(c) for _lo, c in a.ranges], dtype=np.uint16))
    off_b = table(np.array([w for b in a.cls_b for w in words(b)], dtype=np.uint32))
    off_masks = table(np.array(words(a.shift) + words(a.self_loop) + words(a.start), dtype=np.uint32))
    off_follow = table(np.array([w for src, dst, m in a.follow for w in words(src) + words(dst) + [m]], dtype=np.uint32))
    off_accept = table(np.array([w for src, m, p, eo in a.accept for w in words(src) + [m, (first_bit + p) | (int(eo) << 8)]],
                                dtype=np.uint32))
    if a.counters:                   # the counter table is the last of the contiguous tables
        off_ctr = table(np.array([x for pk in a.counters for x in pk], dtype=np.uint32))
        struct.pack_into("<4I", blob, desc_off + 64, len(a.counters), off_ctr, 0, 0)
    struct.pack_into("<16I", blob, desc_off, W, a.n_pos, len(a.cls_b), len(a.ranges), len(a.follow), len(a.accept), a.n_patterns,
                     first_bit, off_ascii, off_lo, off_rck, off_b, off_masks, off_follow, off_accept, len(blob) - off_ascii)
    return desc_off


def _route(patterns: Sequence[Pattern], fits, content: bool = False) -> Tuple[List[int], List[int], Optional[Pna]]:
    """Which of one field's patterns its DFA takes and which go to the position automaton: (dfa indices, nfa indices, the
    automaton of the nfa ones).  The union goes to the DFA whenever it compiles and fits, exactly as without the position
    automaton.  Otherwise every pattern whose DFA is refused (or does not fit) on its own goes to the position automaton, and
    then the patterns with the largest DFAs until the union of the rest fits.  The field's size rule is
    fits(dfa, pna, whole): whether `dfa` fits next to position automaton `pna` (None: alone); `whole` marks the first try.
    `content` selects the body kernel's rules: the union compiled sticky, and the position automaton with counters where the
    plain one is refused (cached_positions(..., counters=True)); head fields keep a plain union and the plain automaton."""
    idx = list(range(len(patterns)))
    try:
        if fits(cached_dfa(patterns, sticky=content), None, True):
            return idx, [], None
    except PatternTooLarge:
        pass
    size: Dict[int, int] = {}
    for i in idx:
        try:
            d = cached_dfa([patterns[i]])
            if fits(d, None, False):
                size[i] = d.n_states
        except PatternTooLarge:
            pass
    dfa = [i for i in idx if i in size]
    while True:
        nfa = [i for i in idx if i not in dfa]
        a = cached_positions([patterns[i] for i in nfa], counters=content)
        if not dfa:
            break
        try:
            if fits(cached_dfa([patterns[i] for i in dfa]), a, False):
                break
        except PatternTooLarge:
            pass
        dfa.remove(max(dfa, key=lambda i: (size[i], i)))
    return dfa, nfa, a


def _body_fits(d: Dfa, a: Optional[Pna], whole: bool) -> bool:
    """Content: the DFA's tables (byte-indexed if small enough, for the union alone) and the position automaton's share the
    body kernel's shared memory."""
    room = BODY_SMEM_LIMIT - (_nfa_table_bytes(a) if a is not None else 0)
    return _table_bytes(d, SMEM_TABLE_LIMIT if whole else 0) <= room


def _head_fits(d: Dfa, a: Optional[Pna], whole: bool) -> bool:
    """Header slots, flags and names: a DFA fits whenever it compiles."""
    return True


def _route_body(patterns: Sequence[Pattern]) -> Tuple[List[int], List[int], Optional[Pna]]:
    return _route(patterns, _body_fits, True)


def _nfa_table_bytes(a: Pna) -> int:
    scratch = bytearray()
    off = serialize_nfa(a, scratch, 0)
    return struct.unpack_from("<I", scratch, off + 60)[0]


class ProgramBuilder:
    def __init__(self):
        self.queries: List[List[Cond]] = []

    def add_query(self, conds: Sequence[Cond]) -> int:
        if len(self.queries) >= 32:
            raise NotImplementedError("at most 32 queries per program")
        self.queries.append(list(conds) if conds else [const(True)])
        return len(self.queries) - 1

    def build(self) -> bytes:
        body = _FieldDfa("content")
        flags = _FieldDfa("flags")
        names = [_FieldDfa("filename"), _FieldDfa("id"), _FieldDfa("hostname"), _FieldDfa("str(timestamp)"), _FieldDfa("str(date)")]
        slots: List[Tuple[str, int, bool]] = []          # (field, mode, empty_if_missing)
        slot_dfas: List[_FieldDfa] = []
        slot_index: Dict[Tuple, int] = {}
        recs: List[Tuple] = []                           # packed cond tuples
        qranges: List[Tuple[int, int]] = []
        head_mask = body_mask = slot_mask = name_mask = 0
        for qi, conds in enumerate(self.queries):
            begin = len(recs)
            for c in conds:
                ref = bit = 0
                if c.kind == C_BODY:
                    bit = body.bit(c.pattern); body_mask |= 1 << qi
                else:
                    head_mask |= 1 << qi
                    if c.kind == C_SLOT:
                        slot_mask |= 1 << qi
                        key = (c.field if c.mode == 1 else c.field.lower(), c.mode, c.empty_if_missing)
                        ref = slot_index.get(key)
                        if ref is None:
                            ref = len(slots)
                            if ref >= 16:
                                raise NotImplementedError("more than 16 distinct header fields in one program")
                            slot_index[key] = ref
                            slots.append(key); slot_dfas.append(_FieldDfa(f"header {c.field}"))
                        bit = slot_dfas[ref].bit(c.pattern)
                    elif c.kind == C_FLAGS:
                        bit = flags.bit(c.pattern)
                    elif c.kind == C_NAME:
                        name_mask |= 1 << qi
                        ref = c.which; bit = names[c.which].bit(c.pattern)
                    elif c.kind == C_CONST:
                        bit = 1 if c.value else 0
                    elif c.kind == C_RECBITS:
                        if not 0 <= c.which < MAX_AUX:
                            raise NotImplementedError("aux column index out of range")
                        ref = c.which
                recs.append((c.kind, ref, bit, 1 if c.negate else 0, c.if_missing, c.op, c.i64, c.set64))
            qranges.append((begin, len(recs)))
        # patterns too large for a field's DFA go to its position automaton; each field's bits are renumbered so that the DFA's
        # outputs come first and the position automaton's follow
        fields = {(C_BODY, 0): body, (C_FLAGS, 0): flags, **{(C_SLOT, k): f for k, f in enumerate(slot_dfas)},
                  **{(C_NAME, k): f for k, f in enumerate(names)}}
        routes = {key: (_route_body(f.patterns) if key[0] == C_BODY else _route(f.patterns, _head_fits)) if f.patterns else ([], [], None)
                  for key, f in fields.items()}
        new_bit = {key: {old: new for new, old in enumerate(dfa + nfa)} for key, (dfa, nfa, _a) in routes.items() if nfa}
        recs = [(kind, ref, new_bit[kind, ref][bit] if (kind, ref) in new_bit else bit, *rest) for kind, ref, bit, *rest in recs]
        body_dfa, body_nfa, pna = routes[C_BODY, 0]

        def head_field(key, direct: int) -> Tuple[int, int]:
            """Serialise a head field: (its DFA's offset, its position automaton's), 0 for a part it does not have."""
            f = fields[key]
            if not f.patterns:
                return 0, 0
            dfa, nfa, a = routes[key]
            if not nfa:
                return serialize_dfa(f.compile(), blob, direct), 0
            off_dfa = serialize_dfa(cached_dfa([f.patterns[i] for i in dfa]), blob, direct) if dfa else 0
            return off_dfa, serialize_nfa(a, blob, len(dfa))

        # small head automata are stored byte-indexed (one lookup per byte in the head kernels) as long as the whole
        # program head still fits the kernels' shared-memory window; otherwise class-indexed (two lookups, smaller)
        for head_direct in (HEAD_DIRECT_LIMIT, 0):
            blob = bytearray(96)
            _pad16(blob)
            off_conds = len(blob)
            for kind, ref, bit, neg, ifm, op, i64, set64 in recs:
                blob.extend(struct.pack("<6B2xqQQ", kind, ref, bit, neg, ifm, op, i64, set64 & 0xFFFFFFFFFFFFFFFF, 0))
            _pad16(blob)
            off_queries = len(blob)
            for a, b in qranges:
                blob.extend(struct.pack("<4I", a, b, 0, 0))
            _pad16(blob)
            for ci, (kind, *_rest, set64) in enumerate(recs):
                if kind == C_FOLDER_SET and set64 >> 64:      # a folder id of 64 or above: the set as a bitmap (fei_prog_cond.off_set_words)
                    n_words = (set64.bit_length() + 31) // 32
                    struct.pack_into("<2I", blob, off_conds + 32 * ci + 24, len(blob), n_words)
                    blob.extend(set64.to_bytes(4 * n_words, "little"))
                    _pad16(blob)
            off_slots = len(blob)
            blob.extend(b"\0" * (16 * len(slots)))
            off_key = 0
            if slots:
                key_pats = [Pattern("regex", "", 0) if mode == 2 else Pattern("exact_equals", f) if mode == 1 else Pattern("equals", f)
                            for f, mode, _e in slots]
                off_key = serialize_dfa(compile_patterns(key_pats), blob)          # only run over the key dictionary (k_key_lut)
                for si, (f, mode, empty) in enumerate(slots):
                    off_val, off_val_nfa = head_field((C_SLOT, si), head_direct)
                    struct.pack_into("<4I", blob, off_slots + 16 * si, mode, off_val, 1 if empty else 0, off_val_nfa)
            off_flags, off_flags_nfa = head_field((C_FLAGS, 0), head_direct)
            off_names, off_name_nfa = zip(*[head_field((C_NAME, k), head_direct) for k in range(len(names))])
            off_head_nfa = 0
            if off_flags_nfa or any(off_name_nfa):         # fei_prog_head_nfa
                _pad16(blob)
                off_head_nfa = len(blob)
                blob.extend(struct.pack("<8I", off_flags_nfa, *off_name_nfa, 0, 0))
            _pad16(blob)
            if len(blob) <= HEAD_SMEM_WINDOW:
                break
        head_bytes = len(blob)               # the content automaton goes last: [0, head_bytes) is what the head kernels stage
        off_nfa = 0
        if not body_nfa:
            off_body = serialize_dfa(body.compile(sticky=True), blob, SMEM_TABLE_LIMIT, tile_bytes=True) if body.patterns else 0
        else:                                # the DFA part class-indexed: k_body_nfa steps one DFA variant
            dfa_pats = [body.patterns[i] for i in body_dfa]
            off_body = serialize_dfa(cached_dfa(dfa_pats), blob, 0, tile_bytes=True) if dfa_pats else 0
            off_nfa = serialize_nfa(pna, blob, len(dfa_pats))
        tb = struct.unpack_from("<I", blob, off_body + 44)[0] if off_body else 0
        if off_nfa:
            tb = tb + struct.unpack_from("<I", blob, off_nfa + 60)[0]
        if tb > BODY_SMEM_LIMIT:
            raise NotImplementedError(f"content automaton needs {tb} bytes of shared memory (limit 220 KiB)")
        _pad16(blob)
        version = VERSION_CTR if pna is not None and pna.counters else VERSION_NFA if any(nfa for _dfa, nfa, _a in routes.values()) else VERSION
        struct.pack_into("<22I", blob, 0, MAGIC, version, len(blob), len(self.queries), len(recs), off_conds,
                         off_queries, len(slots), off_slots, off_key, off_body, off_flags, off_names[0], off_names[1], off_names[2],
                         head_mask, body_mask, slot_mask, name_mask, head_bytes, off_names[3], off_names[4])
        struct.pack_into("<2I", blob, 88, off_nfa, off_head_nfa)
        return bytes(blob)


def content_batch_program(patterns: Sequence[Pattern]) -> bytes:
    """One query per pattern, each a single `content` condition (BASELINE configs[2])."""
    pb = ProgramBuilder()
    for p in patterns:
        pb.add_query([Cond(C_BODY, pattern=p)])
    return pb.build()
