"""Pattern set -> one multi-output UTF-8 byte DFA (host side of the scan kernels).

Everything string-shaped that the reference evaluates per record becomes a DFA run on
the GPU (``fei_b200/csrc/scan.cu``):

* ``matches``           re.search(pattern, value, re.IGNORECASE)            search.py:150-154, filter.py:105
* ``contains`` / ``startswith`` / ``endswith`` / ``=`` / ``!=``   on .lower()ed strings   search.py:148-189
* ``has_tag``           lower().split(","), .strip(), membership             search.py:161-163
* ``has_flag``          str(v2).upper() in flags (ordered substring)         search.py:237-239
* ``> < >= <=``         code-point order of the raw strings                  search.py:227-234

Pipeline: pattern -> code-point NFA (leaf sets taken from CPython's own ``re`` engine /
``str.lower`` so Unicode case rules are exact) -> subset construction over code-point
classes with one character of look-behind / look-ahead context (``^ $ \\A \\Z \\b \\B``,
``(?m)``) -> product with a UTF-8 decoder -> Moore minimisation -> byte classes.

Outputs are Moore masks: ``out[s]`` = patterns whose match is known once the DFA is in
``s``; ``endout[s]`` = patterns that match when the input ends in ``s``.  A value matches
pattern p iff bit p is set in OR(out[s_t]) | endout[s_final].

Not regular / not supported (raise NotImplementedError, never a CPU path): back-references,
look-around, atomic groups / possessive quantifiers, conditional groups.
"""
from __future__ import annotations

import re
from dataclasses import dataclass, field
from typing import Dict, FrozenSet, List, Optional, Sequence, Tuple

import numpy as np

from re import _parser as _P, _compiler as _C, _constants as _K

MAXREPEAT = _K.MAXREPEAT
MAX_CP = 0x10FFFF
_F_I, _F_L, _F_M, _F_S, _F_U, _F_X, _F_A = re.I, re.L, re.M, re.S, re.U, re.X, re.A

RangeSet = Tuple[Tuple[int, int], ...]


class PatternTooLarge(NotImplementedError):
    pass


# --------------------------------------------------------------------------- code point sets
_ALL: Optional[str] = None
_ALL_CP: Optional[np.ndarray] = None


def _all_chars() -> Tuple[str, np.ndarray]:
    global _ALL, _ALL_CP
    if _ALL is None:
        cps = np.concatenate([np.arange(0, 0xD800), np.arange(0xE000, 0x110000)]).astype(np.uint32)
        _ALL = cps.tobytes().decode("utf-32-le")
        _ALL_CP = cps
    return _ALL, _ALL_CP


def _ranges_from_sorted(cps: np.ndarray) -> RangeSet:
    if cps.size == 0:
        return ()
    brk = np.nonzero(np.diff(cps.astype(np.int64)) != 1)[0]
    los = np.concatenate([[0], brk + 1])
    his = np.concatenate([brk, [cps.size - 1]])
    return tuple((int(cps[a]), int(cps[b])) for a, b in zip(los, his))


_leaf_cache: Dict[Tuple, RangeSet] = {}


def regex_leaf_set(node, flags: int) -> RangeSet:
    """Code points a single-character regex node matches, asked of CPython's own engine."""
    key = ("re", repr(node), int(flags) & (_F_I | _F_S | _F_U | _F_A | _F_M))
    hit = _leaf_cache.get(key)
    if hit is not None:
        return hit
    st = _P.State()
    st.flags = flags
    st.str = ""
    rx = _C.compile(_P.SubPattern(st, [node]), flags)
    allc, cps = _all_chars()
    marked = np.frombuffer(rx.sub("\x01", allc).encode("utf-32-le"), dtype=np.uint32)
    sel = marked != cps
    if rx.fullmatch("\x01"):
        sel = sel.copy(); sel[1] = True
    out = _ranges_from_sorted(cps[sel])
    _leaf_cache[key] = out
    return out


_lower_inv: Optional[Dict[int, List[int]]] = None


def _lower_inverse() -> Dict[int, List[int]]:
    """c -> code points x (x != c) whose str.lower() is the single character c."""
    global _lower_inv
    if _lower_inv is None:
        inv: Dict[int, List[int]] = {}
        for x in range(0x110000):
            if 0xD800 <= x <= 0xDFFF:
                continue
            ch = chr(x)
            lo = ch.lower()
            if lo != ch and len(lo) == 1:
                inv.setdefault(ord(lo), []).append(x)
        _lower_inv = inv
    return _lower_inv


def lower_leaf_set(c: int) -> RangeSet:
    """{x : chr(x).lower() == chr(c)} — the characters that become c under str.lower()."""
    key = ("lower", c)
    hit = _leaf_cache.get(key)
    if hit is not None:
        return hit
    xs = list(_lower_inverse().get(c, []))
    if chr(c).lower() == chr(c):
        xs.append(c)
    out = _ranges_from_sorted(np.array(sorted(xs), dtype=np.int64))
    _leaf_cache[key] = out
    return out


_space_set: Optional[RangeSet] = None


def space_set() -> RangeSet:
    """str.strip() / str.isspace() whitespace."""
    global _space_set
    if _space_set is None:
        xs = [x for x in range(0x110000) if not (0xD800 <= x <= 0xDFFF) and chr(x).isspace()]
        _space_set = _ranges_from_sorted(np.array(xs, dtype=np.int64))
    return _space_set


def _uword_set() -> RangeSet:
    return regex_leaf_set((_K.IN, [(_K.CATEGORY, _K.CATEGORY_WORD)]), _F_U)


_AWORD: RangeSet = ((0x30, 0x39), (0x41, 0x5A), (0x5F, 0x5F), (0x61, 0x7A))
_NL: RangeSet = ((0x0A, 0x0A),)
_ANY_ALL: RangeSet = ((0, MAX_CP),)


# --------------------------------------------------------------------------- code point NFA
# assertion codes on epsilon edges
A_BOS, A_BOL, A_EOS, A_EOL, A_WB_U, A_NWB_U, A_WB_A, A_NWB_A, A_NEXTNL = range(1, 10)


class Nfa:
    def __init__(self):
        self.eps: List[List[Tuple[int, int]]] = []      # state -> [(dst, cond)]
        self.chars: List[List[Tuple[int, int]]] = []    # state -> [(leaf_id, dst)]
        self.accept: Dict[int, int] = {}                # state -> pattern id
        self.leaves: List[RangeSet] = []
        self._leaf_ids: Dict[RangeSet, int] = {}
        self.start = self.new()
        self.uses: set = set()
        self.dollar_edges: List[Tuple[int, int]] = []   # non-multiline `$` edges (need the trailing-newline rule)
        self.end_only: set = set()                      # states whose accept only counts at end of input
        self.bound: Dict[Tuple[int, int, int], int] = {}   # counter edges (src, leaf, dst) -> k: `leaf{1,k}` as one edge

    def new(self) -> int:
        self.eps.append([]); self.chars.append([])
        if len(self.eps) > 60000:
            raise PatternTooLarge("pattern set expands to more than 60000 NFA states")
        return len(self.eps) - 1

    def leaf(self, rs: RangeSet) -> int:
        i = self._leaf_ids.get(rs)
        if i is None:
            i = len(self.leaves)
            self.leaves.append(rs)
            self._leaf_ids[rs] = i
        return i

    def e(self, a: int, b: int, cond: int = 0) -> None:
        self.eps[a].append((b, cond))
        if cond:
            self.uses.add(cond)

    def c(self, a: int, rs: RangeSet, b: int) -> None:
        self.chars[a].append((self.leaf(rs), b))

    def add_trailing_newline_rule(self) -> None:
        """Non-multiline `$` also matches just before a newline that ends the string (two characters of
        look-ahead).  Modelled with two shadow copies of the automaton: level 1 = "continuing from a `$`
        taken before a '\\n', valid only if that newline is the last character", level 2 = "that newline has
        been consumed; valid only at end of input".  Level-2 accepts count at end of input only."""
        if not self.dollar_edges:
            return
        N = len(self.eps)
        nl = self.leaf(_NL)
        base_eps = [list(e) for e in self.eps]
        base_chars = [list(c) for c in self.chars]
        base_accept = dict(self.accept)
        for _ in range(2 * N):
            self.new()
        for q in range(N):
            for d, cond in base_eps[q]:
                self.eps[q + N].append((d + N, cond))
                self.eps[q + 2 * N].append((d + 2 * N, cond))
            for leaf_id, d in base_chars[q]:
                if any(lo <= 0x0A <= hi for lo, hi in self.leaves[leaf_id]):
                    self.chars[q + N].append((nl, d + 2 * N))          # consumes the final newline itself
            p = base_accept.get(q)
            if p is not None:
                acc2 = self.new()
                self.accept[acc2] = p; self.end_only.add(acc2)
                self.chars[q + N].append((nl, acc2))                   # matched before the final newline
                self.accept[q + 2 * N] = p; self.end_only.add(q + 2 * N)
        for a, b in self.dollar_edges:
            self.eps[a].append((b + N, A_NEXTNL))
            self.eps[a + N].append((b + N, A_NEXTNL))
        self.uses.add(A_NEXTNL)


def _single_leaf(p, flags: int):
    """(leaf node, its flags) when repeat body `p` is one character leaf, possibly inside groups or inline-flag groups."""
    while len(p) == 1:
        op, av = p[0]
        if op in (_K.LITERAL, _K.NOT_LITERAL, _K.ANY, _K.IN):
            return p[0], flags
        if op is not _K.SUBPATTERN:
            return None
        _group, add, dele, p = av
        flags = (flags | add) & ~dele
    return None


def _countable(node, flags: int) -> bool:
    """A repeat a counter can hold: `C{lo,hi}` with a finite hi > lo and one character leaf C."""
    op, av = node
    if op not in (_K.MAX_REPEAT, _K.MIN_REPEAT):
        return False
    lo, hi, p = av
    return hi is not MAXREPEAT and hi != MAXREPEAT and hi > lo and _single_leaf(p, flags) is not None


def _countable_repeats(items, flags: int, out: list) -> list:
    """Countable repeats of an AST in a fixed depth-first order: [(node, hi - lo)].  Repeats inside a countable one are not
    visited (its body is a single character)."""
    for node in items:
        op, av = node
        if _countable(node, flags):
            out.append((node, av[1] - av[0]))
        elif op is _K.SUBPATTERN:
            _countable_repeats(av[3], (flags | av[1]) & ~av[2], out)
        elif op is _K.BRANCH:
            for alt in av[1]:
                _countable_repeats(alt, flags, out)
        elif op in (_K.MAX_REPEAT, _K.MIN_REPEAT):
            _countable_repeats(av[2], flags, out)
    return out


class _RegexBuilder:
    """re._parser AST -> NFA fragment (Thompson construction).  `counted`: ids of the countable repeat nodes that become one
    counter edge each (compile_positions_counted) instead of hi expanded copies."""

    def __init__(self, nfa: Nfa, counted: FrozenSet[int] = frozenset()):
        self.n = nfa
        self.counted = counted

    def seq(self, items, flags: int, a: int) -> int:
        cur = a
        for node in items:
            cur = self.node(node, flags, cur)
        return cur

    def node(self, node, flags: int, a: int) -> int:
        n = self.n
        op, av = node
        if op in (_K.LITERAL, _K.NOT_LITERAL, _K.ANY, _K.IN):
            b = n.new()
            n.c(a, regex_leaf_set(node, flags), b)
            return b
        if op is _K.SUBPATTERN:
            _group, add, dele, p = av
            return self.seq(p, (flags | add) & ~dele, a)
        if op is _K.BRANCH:
            b = n.new()
            for alt in av[1]:
                s = n.new(); n.e(a, s)
                n.e(self.seq(alt, flags, s), b)
            return b
        if op in (_K.MAX_REPEAT, _K.MIN_REPEAT):
            lo, hi, p = av
            cur = a
            if id(node) in self.counted:             # lo copies, then C{0,hi-lo} as the epsilon bypass and one counter edge
                if lo > 1000:
                    raise PatternTooLarge("repeat count above 1000")
                for _ in range(lo):
                    cur = self.seq(p, flags, cur)
                leaf, lflags = _single_leaf(p, flags)
                t = n.new(); out = n.new()
                rs = regex_leaf_set(leaf, lflags)
                n.c(cur, rs, t)
                n.bound[(cur, n.leaf(rs), t)] = hi - lo
                n.e(cur, out); n.e(t, out)
                return out
            if lo > 1000 or (hi is not MAXREPEAT and hi > 1000):
                raise PatternTooLarge("repeat count above 1000")
            for _ in range(lo):
                cur = self.seq(p, flags, cur)
            if hi is MAXREPEAT or hi == MAXREPEAT:
                loop = n.new(); n.e(cur, loop)
                end = self.seq(p, flags, loop)
                n.e(end, loop)
                out = n.new(); n.e(loop, out)
                return out
            out = n.new(); n.e(cur, out)
            for _ in range(hi - lo):
                cur = self.seq(p, flags, cur)
                n.e(cur, out)
            return out
        if op is _K.AT:
            b = n.new()
            multi = bool(flags & _F_M)
            ascii_ = bool(flags & _F_A)
            cond = {
                _K.AT_BEGINNING: A_BOL if multi else A_BOS,
                _K.AT_BEGINNING_STRING: A_BOS,
                _K.AT_END: A_EOL if multi else A_EOS,     # + the trailing-newline rule, see Nfa.add_trailing_newline_rule
                _K.AT_END_STRING: A_EOS,
                _K.AT_BOUNDARY: A_WB_A if ascii_ else A_WB_U,
                _K.AT_NON_BOUNDARY: A_NWB_A if ascii_ else A_NWB_U,
            }.get(av)
            if cond is None:
                raise NotImplementedError(f"regex assertion {av} is not supported on the GPU")
            n.e(a, b, cond)
            if av == _K.AT_END and not multi:
                n.dollar_edges.append((a, b))
            return b
        if op in (_K.ASSERT, _K.ASSERT_NOT):
            raise NotImplementedError("look-ahead / look-behind is not regular: not supported on the GPU")
        if op in (_K.GROUPREF, _K.GROUPREF_EXISTS):
            raise NotImplementedError("back-references are not regular: not supported on the GPU")
        if op in (getattr(_K, "ATOMIC_GROUP", None), getattr(_K, "POSSESSIVE_REPEAT", None)):
            raise NotImplementedError("atomic groups / possessive quantifiers are not supported on the GPU")
        raise NotImplementedError(f"regex construct {op} is not supported on the GPU")


@dataclass
class Pattern:
    """One predicate over a string value.  kind:
    regex(text, flags) | contains | startswith | endswith | equals | has_tag (all via str.lower()),
    exact_contains | exact_equals (no folding) | cmp_gt | cmp_ge | cmp_lt | cmp_le (raw code-point order)."""
    kind: str
    text: str
    flags: int = 0


_IDOT: RangeSet = ((0x130, 0x130),)


def _lit_chain(n: Nfa, a: int, text: str, lowered: bool, end_half: bool = False, start_half_from: Optional[int] = None) -> int:
    """States a -> ... -> end that consume `text`.  lowered: the VALUE is read through str.lower().  lower() is per character
    except U+0130, which becomes the two characters 'i' + U+0307: one input character then advances the needle by two
    ('i', U+0307), by its last one (needle ends in 'i' and may end inside the expansion: `end_half`, for contains /
    startswith) or lets a match begin at the combining dot (`start_half_from` = the state an unanchored match starts from,
    for contains / endswith).  (Capital sigma's final-form rule is the one context-dependent case left: the host layer refuses
    needles containing a sigma on corpora that hold U+03A3.)"""
    states = [a]
    for ch in text:
        b = n.new()
        n.c(states[-1], lower_leaf_set(ord(ch)) if lowered else ((ord(ch), ord(ch)),), b)
        states.append(b)
    if lowered and text:
        for p in range(len(text) - 1):
            if text[p] == "i" and text[p + 1] == "\u0307":
                n.c(states[p], _IDOT, states[p + 2])
        if end_half and text[-1] == "i":
            n.c(states[-2], _IDOT, states[-1])
        if start_half_from is not None and text[0] == "\u0307":
            n.c(start_half_from, _IDOT, states[1])
    return states[-1]


_SIGMA = 0x3A3
_PH = "\U0010FFFE"        # placeholder (a noncharacter) that marks a needle sigma inside the plain fragment
_case_classes: Optional[Tuple[RangeSet, RangeSet]] = None


def _case_class_sets() -> Tuple[RangeSet, RangeSet]:
    """(case-ignorable, cased-and-not-ignorable) code point sets exactly as str.lower()'s final-sigma rule sees them
    (Objects/unicodeobject.c handle_capital_sigma), obtained by asking str.lower() itself:
    'A' + c + 'Σ' lowers to a final sigma iff c is case-ignorable or cased; c + 'Σ' iff c is cased and not ignorable."""
    global _case_classes
    if _case_classes is None:
        ign, cased = [], []
        for x in range(0x110000):
            if 0xD800 <= x <= 0xDFFF:
                continue
            ch = chr(x)
            alone = (ch + "Σ").lower()[-1] == "ς"
            after = ("A" + ch + "Σ").lower()[-1] == "ς"
            if alone:
                cased.append(x)
            elif after:
                ign.append(x)
        _case_classes = (_ranges_from_sorted(np.array(ign, dtype=np.int64)), _ranges_from_sorted(np.array(cased, dtype=np.int64)))
    return _case_classes


def _rs_and(a: RangeSet, b: RangeSet) -> RangeSet:
    out = []
    i = j = 0
    while i < len(a) and j < len(b):
        lo, hi = max(a[i][0], b[j][0]), min(a[i][1], b[j][1])
        if lo <= hi:
            out.append((lo, hi))
        if a[i][1] < b[j][1]:
            i += 1
        else:
            j += 1
    return tuple(out)


def _rs_not(a: RangeSet) -> RangeSet:
    out = []
    prev = 0
    for lo, hi in a:
        if lo > prev:
            out.append((prev, lo - 1))
        prev = hi + 1
    if prev <= MAX_CP:
        out.append((prev, MAX_CP))
    return tuple(out)


def _add_sigma_exact(n: Nfa, pid: int, pat: Pattern) -> None:
    """Lower-casing pattern whose needle holds a sigma, exact over text with capital sigmas.  str.lower() turns U+03A3 into the
    final form (U+03C2) iff it is preceded by a cased letter and not followed by one, case-ignorable characters skipped on both
    sides.  The pattern's plain automaton is multiplied with that rule: every thread carries B = 'the text so far ends in a cased
    letter (+ ignorables)' and a pending obligation about what must follow a capital sigma it consumed -- F (read as final: no cased
    letter may follow) or M (read as medial: one must).  Reading a capital sigma as a needle character forks the two readings; the
    wrong one dies when the following characters contradict it."""
    f = Nfa()
    add_pattern(f, 0, Pattern(pat.kind, pat.text.replace("σ", _PH + "s").replace("ς", _PH + "f"), pat.flags), _plain=True)   # placeholders, replaced below
    ign, cased = _case_class_sets()
    sig: RangeSet = ((_SIGMA, _SIGMA),)
    not_sig = _rs_not(sig)
    classes = {"I": _rs_and(ign, not_sig), "C": _rs_and(cased, not_sig), "O": _rs_and(_rs_and(_rs_not(ign), _rs_not(cased)), not_sig)}
    prod: Dict[Tuple[int, int, str], int] = {}

    def P(q: int, b: int, ob: str) -> int:
        k = (q, b, ob)
        v = prod.get(k)
        if v is None:
            v = prod[k] = n.new()
        return v

    def resolve(ob: str, cls: str) -> Optional[str]:
        if ob == "F":
            return {"I": "F", "C": None, "O": ""}[cls]
        if ob == "M":
            return {"I": "M", "C": "", "O": None}[cls]
        return ""

    def next_b(b: int, cls: str) -> int:
        return b if cls == "I" else 1 if cls == "C" else 0

    # the fragment was built with two-character placeholders for the sigmas: (_PH, 's') = medial sigma, (_PH, 'f') = final sigma.
    # Collapse each placeholder pair into one edge with a marker.
    nul: RangeSet = ((ord(_PH), ord(_PH)),)
    edges: Dict[int, List[Tuple[Any, int]]] = {q: [] for q in range(len(f.chars))}
    for q in range(len(f.chars)):
        for leaf_id, d in f.chars[q]:
            S = f.leaves[leaf_id]
            if S == nul:                                          # first half of a placeholder: look through to its second half
                for leaf2, d2 in f.chars[d]:
                    S2 = f.leaves[leaf2]
                    edges[q].append(("sigma_medial" if any(lo <= ord("s") <= hi for lo, hi in S2) else "sigma_final", d2))
            else:
                edges[q].append((S, d))
    mid_states = {d for q in range(len(f.chars)) for leaf_id, d in f.chars[q] if f.leaves[leaf_id] == nul}
    terminal = {a for a in f.accept if not f.chars[a]}
    for q in range(len(f.chars)):
        if q in mid_states:
            continue
        for b in (0, 1):
            for ob in ("", "F", "M"):
                src = None
                for S, d in edges[q]:
                    if src is None:
                        src = P(q, b, ob)
                    if isinstance(S, str):                        # a needle sigma
                        want_final = S == "sigma_final"
                        lit: RangeSet = ((0x3C2, 0x3C2),) if want_final else ((0x3C3, 0x3C3),)       # the lower-case letter itself (cased, not ignorable)
                        r = resolve(ob, "C")
                        if r is not None:
                            n.c(src, lit, P(d, 1, r))
                            if want_final and b:                  # capital sigma read as final
                                n.c(src, sig, P(d, 1, "F"))
                            if not want_final:                    # capital sigma read as medial (certainly medial without a cased letter before it)
                                n.c(src, sig, P(d, 1, "M" if b else ""))
                        continue
                    for cls, cset in classes.items():
                        part = _rs_and(S, cset)
                        r = resolve(ob, cls)
                        if part and r is not None:
                            n.c(src, part, P(d, next_b(b, cls), r))
                    if any(lo <= _SIGMA <= hi for lo, hi in S):    # a capital sigma whose lowered form this edge does not care about
                        r = resolve(ob, "C")
                        if r is not None:
                            n.c(src, sig, P(d, 1, r))
                for d, cond in f.eps[q]:
                    if src is None:
                        src = P(q, b, ob)
                    n.e(src, P(d, b, ob), cond)
                    if cond:
                        n.uses.add(cond)
                if q in f.accept:
                    here = P(q, b, ob)
                    if ob == "":
                        n.accept[here] = pid
                        if q in f.end_only:
                            n.end_only.add(here)
                    elif ob == "F":                               # fine if the text ends here
                        n.accept[here] = pid; n.end_only.add(here)
                    if q in terminal and ob:                      # matched, the last sigma's reading still to be confirmed by what follows
                        for cls, cset in classes.items():
                            r = resolve(ob, cls)
                            if r is not None:
                                n.c(here, cset, P(q, next_b(b, cls), r))
                        r = resolve(ob, "C")
                        if r is not None:
                            n.c(here, sig, P(q, 1, r))
    n.e(n.start, P(f.start, 0, ""))


def add_pattern(n: Nfa, pid: int, pat: Pattern, _plain: bool = False, counted: Sequence[int] = ()) -> None:
    """Attach pattern `pid` to the union NFA.  `n.start` is the global start (position 0 only).  counted (regex only): indices
    into _countable_repeats of the pattern's AST of the repeats built as counter edges."""
    k = pat.kind
    if not _plain and k in ("contains", "startswith", "endswith", "equals", "has_tag") and ("\u03c3" in pat.text or "\u03c2" in pat.text):
        _add_sigma_exact(n, pid, pat)
        return
    if k == "regex":
        ast = _P.parse(pat.text, pat.flags)           # re.error propagates to the caller
        flags = ast.state.flags
        if flags & _F_L:
            raise NotImplementedError("re.LOCALE")
        u = n.new()                                   # unanchored search: every position may start a match
        n.e(n.start, u)
        n.c(u, _ANY_ALL, u)
        s = n.new(); n.e(u, s)
        ids = frozenset()
        if counted:
            reps = _countable_repeats(ast.data, flags, [])
            ids = frozenset(id(reps[i][0]) for i in counted)
        end = _RegexBuilder(n, ids).seq(ast.data, flags, s)
        n.accept[end] = pid
        return
    if k in ("contains", "exact_contains"):
        lowered = k == "contains"
        u = n.new(); n.e(n.start, u); n.c(u, _ANY_ALL, u)
        end = _lit_chain(n, u, pat.text, lowered, end_half=True, start_half_from=u)
        n.accept[end] = pid
        return
    if k == "startswith":
        end = _lit_chain(n, n.start, pat.text, True, end_half=True)
        n.accept[end] = pid
        return
    if k == "endswith":
        u = n.new(); n.e(n.start, u); n.c(u, _ANY_ALL, u)
        end = _lit_chain(n, u, pat.text, True, start_half_from=u)
        acc = n.new(); n.e(end, acc, A_EOS)
        n.accept[acc] = pid
        return
    if k in ("equals", "exact_equals"):
        end = _lit_chain(n, n.start, pat.text, k == "equals")
        acc = n.new(); n.e(end, acc, A_EOS)
        n.accept[acc] = pid
        return
    if k == "has_tag":
        t = pat.text
        if "," in t or t != t.strip():
            return                                    # can never equal a stripped comma-free piece
        ws = space_set()
        comma = ((0x2C, 0x2C),)
        u = n.new(); n.e(n.start, u); n.c(u, _ANY_ALL, u)
        a = n.new(); n.e(n.start, a); n.c(u, comma, a)   # piece start: position 0 or right after ','
        n.c(a, ws, a)
        b = _lit_chain(n, a, t, True)
        n.c(b, ws, b)
        acc = n.new()
        n.e(b, acc, A_EOS)
        n.c(b, comma, acc)
        n.accept[acc] = pid
        return
    if k in ("cmp_gt", "cmp_ge", "cmp_lt", "cmp_le"):
        t = pat.text
        gt = n.new(); n.c(gt, _ANY_ALL, gt)
        lt = n.new(); n.c(lt, _ANY_ALL, lt)
        cur = n.start
        acc = n.new()
        for ch in t:
            c = ord(ch)
            nxt = n.new()
            if c > 0:
                n.c(cur, ((0, c - 1),), lt)
            n.c(cur, ((c, c),), nxt)
            if c < MAX_CP:
                n.c(cur, ((c + 1, MAX_CP),), gt)
            if k in ("cmp_lt", "cmp_le"):
                n.e(cur, acc, A_EOS)                  # value is a proper prefix of the operand: value < operand
            cur = nxt
        n.c(cur, _ANY_ALL, gt)                        # operand is a proper prefix of the value: value > operand
        if k in ("cmp_ge", "cmp_le"):
            n.e(cur, acc, A_EOS)                      # equal
        n.e(gt if k in ("cmp_gt", "cmp_ge") else lt, acc, A_EOS)
        n.accept[acc] = pid
        return
    raise ValueError(f"unknown pattern kind {k!r}")


# --------------------------------------------------------------------------- classes
def _partition(leaves: Sequence[RangeSet]) -> Tuple[np.ndarray, List[FrozenSet[int]]]:
    """Elementary intervals of [0, 0x1FFFFF] -> class ids.  Returns (bounds, class_of_interval, members)."""
    cuts = {0, 0x200000}
    for rs in leaves:
        for lo, hi in rs:
            cuts.add(lo); cuts.add(hi + 1)
    bounds = np.array(sorted(cuts), dtype=np.int64)
    nint = len(bounds) - 1
    sig = [0] * nint                                     # python ints as bitsets over leaves
    for li, rs in enumerate(leaves):
        for lo, hi in rs:
            a = int(np.searchsorted(bounds, lo)); b = int(np.searchsorted(bounds, hi + 1))
            bit = 1 << li
            for j in range(a, b):
                sig[j] |= bit
    ids: Dict[int, int] = {}
    cls_of = np.zeros(nint, dtype=np.int32)
    members: List[int] = []
    for j, s in enumerate(sig):
        if s not in ids:
            ids[s] = len(ids); members.append(s)
        cls_of[j] = ids[s]
    return bounds, cls_of, members


@dataclass
class Dfa:
    trans: np.ndarray            # [n_states, 256] int32 (byte level)
    out: np.ndarray              # [n_states] uint32
    endout: np.ndarray           # [n_states] uint32
    start: int
    n_patterns: int
    cls: np.ndarray = field(default=None)     # [256] uint8 byte classes
    ctrans: np.ndarray = field(default=None)  # [n_states, n_cls] int32
    sticky_state: int = -2                    # >= 0: absorbing "matched" state of a sticky DFA; -1: sticky, can never match

    @property
    def n_states(self) -> int:
        return self.trans.shape[0]

    def run(self, data: bytes) -> int:
        """Host simulation (tests only): mask of matching patterns for `data`."""
        s = self.start
        acc = int(self.out[s])
        t = self.trans
        for b in data:
            s = int(t[s, b])
            acc |= int(self.out[s])
        return acc | int(self.endout[s])


def compile_patterns(patterns: Sequence[Pattern], max_states: int = 30000, sticky: bool = False) -> Dfa:
    """sticky=True (single pattern only): once the pattern has matched the automaton parks in one absorbing
    state whose `endout` carries the verdict, so a scan kernel needs no per-byte accept bookkeeping and can
    stop reading a record early."""
    if len(patterns) > 32:
        raise ValueError("at most 32 patterns per DFA")
    n = Nfa()
    for pid, p in enumerate(patterns):
        add_pattern(n, pid, p)
    n.add_trailing_newline_rule()
    d = _determinize(n, len(patterns), max_states)
    if sticky and len(patterns) == 1:
        d = make_sticky(d)
    return d


def make_sticky(d: Dfa) -> Dfa:
    acc = np.nonzero(d.out != 0)[0]
    T = d.trans.copy(); out = d.out.copy(); endout = d.endout.copy()
    T[acc, :] = acc[:, None]                      # self-loops: a match can never be lost again
    endout[acc] |= out[acc]
    out[:] = 0                                    # the verdict is read from endout only
    T, out, endout, start = _minimize(T, out, endout, d.start)
    nd = Dfa(trans=T, out=out, endout=endout, start=start, n_patterns=d.n_patterns)
    _byte_classes(nd)
    absorbing = np.nonzero((T == np.arange(T.shape[0])[:, None]).all(axis=1) & (endout != 0))[0]
    nd.sticky_state = int(absorbing[0]) if absorbing.size else -1
    return nd


def _determinize(n: Nfa, npat: int, max_states: int) -> Dfa:
    uses = n.uses
    need_nl = A_BOL in uses or A_EOL in uses or A_NEXTNL in uses
    need_uw = A_WB_U in uses or A_NWB_U in uses
    need_aw = A_WB_A in uses or A_NWB_A in uses
    leaves = list(n.leaves)
    ctx_leaf = {}
    if need_nl:
        ctx_leaf["nl"] = len(leaves); leaves.append(_NL)
    if need_uw:
        ctx_leaf["uw"] = len(leaves); leaves.append(_uword_set())
    if need_aw:
        ctx_leaf["aw"] = len(leaves); leaves.append(_AWORD)
    bounds, cls_of, members = _partition(leaves)
    ncls = len(members)
    # per class: context bits (nl, uword, aword) and leaf membership
    def bit(m, name):
        return (m >> ctx_leaf[name]) & 1 if name in ctx_leaf else 0
    cls_ctx = [(bit(m, "nl"), bit(m, "uw"), bit(m, "aw")) for m in members]
    START_CTX, END_CTX = (2, 0, 0), (3, 0, 0)        # first component: 0/1 = nl bit, 2 = start of text, 3 = end
    nleaf = len(n.leaves)
    # move table per NFA state: class -> list of dst
    moves: List[Dict[int, List[int]]] = []
    for s in range(len(n.chars)):
        d: Dict[int, List[int]] = {}
        for leaf_id, dst in n.chars[s]:
            bitv = 1 << leaf_id
            for c in range(ncls):
                if members[c] & bitv:
                    d.setdefault(c, []).append(dst)
        moves.append(d)

    def cond_ok(cond: int, prev, nxt) -> bool:
        if cond == A_BOS:
            return prev[0] == 2
        if cond == A_BOL:
            return prev[0] == 2 or prev[0] == 1
        if cond == A_EOS:
            return nxt[0] == 3
        if cond == A_EOL:
            return nxt[0] == 3 or nxt[0] == 1
        if cond == A_NEXTNL:
            return nxt[0] == 1
        if prev[0] == 2 and nxt[0] == 3:
            return False                                 # empty input: neither \b nor \B matches (CPython 3.12)
        k = 1 if cond in (A_WB_U, A_NWB_U) else 2
        pw = prev[k] if prev[0] != 2 else 0
        nw = nxt[k] if nxt[0] != 3 else 0
        return (pw != nw) if cond in (A_WB_U, A_WB_A) else (pw == nw)

    eps = n.eps
    any_cond = bool(uses)
    clo_cache: Dict[Tuple, FrozenSet[int]] = {}

    def closure(states: FrozenSet[int], prev, nxt) -> FrozenSet[int]:
        key = (states, prev, nxt) if any_cond else states
        hit = clo_cache.get(key)
        if hit is not None:
            return hit
        seen = set(states)
        stack = list(states)
        while stack:
            s = stack.pop()
            for dst, cond in eps[s]:
                if dst not in seen and (cond == 0 or cond_ok(cond, prev, nxt)):
                    seen.add(dst); stack.append(dst)
        out = frozenset(seen)
        clo_cache[key] = out
        return out

    acc = n.accept
    end_only = n.end_only

    def mask_of(states, at_end: bool = False) -> int:
        m = 0
        for s in states:
            p = acc.get(s)
            if p is not None and (at_end or s not in end_only):
                m |= 1 << p
        return m

    track = (need_nl, need_uw, need_aw)

    def norm_ctx(c):           # keep only the context bits some assertion reads (fewer DFA states)
        return (c[0] if track[0] else 0, c[1] if track[1] else 0, c[2] if track[2] else 0)

    # Matches that do not depend on the next character are reported eagerly, as a function of the
    # state alone (Moore output without state splitting: a plain literal set stays an Aho-Corasick
    # automaton).  Only accepts behind a look-ahead assertion ($, \Z, \b, \B) are delayed to
    # the next transition and folded into the target state's identity.
    eager_cache: Dict[Tuple, int] = {}

    def eager(states: FrozenSet[int], prev) -> int:
        key = (states, prev)
        hit = eager_cache.get(key)
        if hit is not None:
            return hit
        seen = set(states)
        stack = list(states)
        while stack:
            s = stack.pop()
            for dst, cond in eps[s]:
                if dst in seen:
                    continue
                if cond == 0 or (cond == A_BOS and prev[0] == 2) or (cond == A_BOL and prev[0] in (1, 2)):
                    seen.add(dst); stack.append(dst)
        m = mask_of(seen)
        eager_cache[key] = m
        return m

    zero_ctx = (0, 0, 0)
    start_prev = START_CTX if any_cond else zero_ctx
    start_set = frozenset([n.start])
    start_key = (start_set, start_prev, eager(start_set, start_prev))
    index: Dict[Tuple, int] = {start_key: 0}
    order = [start_key]
    rows: List[List[int]] = []
    i = 0
    while i < len(order):
        S, prev, _m = order[i]
        eg = eager(S, prev)
        row = [0] * ncls
        for c in range(ncls):
            nxt_ctx = cls_ctx[c]
            C = closure(S, prev, nxt_ctx)
            delayed = mask_of(C) & ~eg
            T = set()
            for s in C:
                d = moves[s].get(c)
                if d:
                    T.update(d)
            Tf = frozenset(T)
            nprev = norm_ctx(nxt_ctx) if any_cond else zero_ctx
            key = (Tf, nprev, delayed | eager(Tf, nprev))
            j = index.get(key)
            if j is None:
                j = len(order)
                if j >= max_states:
                    raise PatternTooLarge(f"code-point DFA exceeds {max_states} states")
                index[key] = j; order.append(key)
            row[c] = j
        rows.append(row)
        i += 1
    ncp = len(order)
    cp_trans = np.array(rows, dtype=np.int32).reshape(ncp, ncls)
    cp_out = np.array([k[2] for k in order], dtype=np.uint32)
    cp_end = np.array([mask_of(closure(k[0], k[1], END_CTX), at_end=True) for k in order], dtype=np.uint32)
    # the mask emitted on entry is also valid at the end (it was already counted); fold nothing more
    return _to_bytes(cp_trans, cp_out, cp_end, bounds, cls_of, ncls, npat)


# --------------------------------------------------------------------------- UTF-8 product
def _to_bytes(cp_trans, cp_out, cp_end, bounds, cls_of, ncls, npat) -> Dfa:
    """Code-point DFA -> byte DFA.  Each code-point state becomes a byte state; multi-byte
    characters get intermediate decoder states that are shared between all code-point states
    with the same (remaining bytes, target segmentation) signature, so the result stays close
    to minimal even with Unicode classes (\\w has ~770 ranges)."""
    ncp = cp_trans.shape[0]
    rows: List[Optional[np.ndarray]] = [None] * ncp
    sig2id: Dict[Tuple, int] = {}
    DEAD = -1                                            # patched to the sink id at the end
    cont = np.arange(0x80, 0xC0)

    def targets_at(tgt: np.ndarray, cps: np.ndarray) -> np.ndarray:
        return tgt[np.searchsorted(bounds, cps, side="right") - 1]

    def segs(tgt: np.ndarray, lo: int, hi: int) -> Tuple[Tuple[int, int], ...]:
        a = int(np.searchsorted(bounds, lo, side="right") - 1)
        b = int(np.searchsorted(bounds, hi, side="right") - 1)
        vals = tgt[a:b + 1]
        if a == b or not np.any(vals[1:] != vals[:-1]):
            return ((0, int(vals[0])),)
        starts = np.concatenate([[0], np.nonzero(vals[1:] != vals[:-1])[0] + 1])
        return tuple((max(int(bounds[a + st]), lo) - lo, int(vals[st])) for st in starts)

    def node(tgt: np.ndarray, lo: int, k: int, sg=None, bmin: int = 0x80, bmax: int = 0xBF) -> int:
        """Byte state that still has to read k continuation bytes of a character in lo..lo+64^k-1.
        bmin/bmax restrict the next byte (overlong forms, surrogates and > U+10FFFF go to the sink)."""
        step = 64 ** (k - 1)
        if sg is None:
            sg = segs(tgt, lo + (bmin - 0x80) * step, lo + (bmax - 0x80 + 1) * step - 1)
        key = (k, sg, bmin, bmax)
        j = sig2id.get(key)
        if j is not None:
            return j
        j = len(rows)
        sig2id[key] = j
        rows.append(None)
        if len(rows) > 60000:
            raise PatternTooLarge("byte automaton exceeds 60000 states")
        row = np.full(256, DEAD, dtype=np.int64)
        if len(sg) == 1:
            t = sg[0][1]
            row[bmin:bmax + 1] = t if k == 1 else node(tgt, lo + (bmin - 0x80) * step, k - 1, sg)
        elif k == 1:
            row[bmin:bmax + 1] = targets_at(tgt, lo + (cont[bmin - 0x80:bmax - 0x80 + 1] - 0x80))
        else:
            for b in range(bmin, bmax + 1):
                row[b] = node(tgt, lo + (b - 0x80) * step, k - 1)
        rows[j] = row
        return j

    ascii_cps = np.arange(0x80)
    for S in range(ncp):
        tgt = cp_trans[S][cls_of].astype(np.int64)       # target state per elementary interval
        row = np.full(256, DEAD, dtype=np.int64)
        row[:0x80] = targets_at(tgt, ascii_cps)
        for b in range(0xC2, 0xE0):
            row[b] = node(tgt, (b & 0x1F) << 6, 1)
        for b in range(0xE0, 0xF0):
            row[b] = node(tgt, (b & 0x0F) << 12, 2, None, 0xA0 if b == 0xE0 else 0x80, 0x9F if b == 0xED else 0xBF)
        for b in range(0xF0, 0xF5):
            row[b] = node(tgt, (b & 0x07) << 18, 3, None, 0x90 if b == 0xF0 else 0x80, 0x8F if b == 0xF4 else 0xBF)
        rows[S] = row
    nstates = len(rows) + 1
    sink = nstates - 1
    T = np.stack(rows + [np.full(256, DEAD, dtype=np.int64)])
    T[T == DEAD] = sink
    out = np.zeros(nstates, dtype=np.uint32); endout = np.zeros(nstates, dtype=np.uint32)
    out[:ncp] = cp_out; endout[:ncp] = cp_end
    T, out, endout, start = _minimize(T.astype(np.int32), out, endout, 0)
    d = Dfa(trans=T, out=out, endout=endout, start=start, n_patterns=npat)
    _byte_classes(d)
    return d


def _minimize(T: np.ndarray, out: np.ndarray, endout: np.ndarray, start: int):
    n = T.shape[0]
    # collapse identical columns first (cheaper refinement): columns are grouped by a 64-bit hash, then checked exactly
    with np.errstate(over="ignore"):
        rmult = (np.arange(1, n + 1, dtype=np.uint64) * np.uint64(0xD6E8FEB86659FD93)) | np.uint64(1)
        colh = (T.astype(np.uint64) * rmult[:, None]).sum(axis=0, dtype=np.uint64)
    _, col_first, col_inv = np.unique(colh, return_index=True, return_inverse=True)
    if not np.array_equal(T, T[:, col_first[col_inv.reshape(-1)]]):      # two different columns with one hash: compare columns themselves
        _, col_first, col_inv = np.unique(T, axis=1, return_index=True, return_inverse=True)
    Tc = T[:, np.sort(col_first)]
    key = out.astype(np.int64) << 32 | endout.astype(np.int64)
    _, block = np.unique(key, return_inverse=True)
    block = block.reshape(-1)
    nblocks = int(block.max()) + 1
    # Moore refinement on 64-bit hashes of the signature rows (a 1-D unique per round instead of a row-wise one); a hash
    # collision could only merge two different signatures, which the exact check below would expose
    mult = (np.arange(1, Tc.shape[1] + 2, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)) | np.uint64(1)
    with np.errstate(over="ignore"):
        while True:
            h = block.astype(np.uint64) * mult[0] + (block[Tc].astype(np.uint64) * mult[None, 1:]).sum(axis=1, dtype=np.uint64)
            _, newblock = np.unique(h, return_inverse=True)
            newblock = newblock.reshape(-1)
            nb = int(newblock.max()) + 1
            block = newblock
            if nb == nblocks:
                break
            nblocks = nb
    rep0 = np.full(nblocks, n, dtype=np.int64)
    np.minimum.at(rep0, block, np.arange(n))
    sig = np.concatenate([key[:, None], block[Tc]], axis=1)
    if not np.array_equal(sig, sig[rep0[block]]):            # never seen; exact row-wise refinement from scratch
        _, block = np.unique(key, return_inverse=True)
        block = block.reshape(-1)
        nblocks = int(block.max()) + 1
        while True:
            sig = np.concatenate([block[:, None], block[Tc]], axis=1)
            _, newblock = np.unique(sig, axis=0, return_inverse=True)
            nb = int(newblock.max()) + 1
            block = newblock.reshape(-1)
            if nb == nblocks:
                break
            nblocks = nb
    # representative per block, block of start first
    # stable numbering by first occurrence, with the start state's block as 0
    first_idx = np.full(nblocks, n, dtype=np.int64)
    np.minimum.at(first_idx, block, np.arange(n))
    ranks = np.argsort(first_idx, kind="stable")
    # move start's block to the front
    sb = int(block[start])
    ranks = np.concatenate([[sb], ranks[ranks != sb]])
    new_id = np.empty(nblocks, dtype=np.int64)
    new_id[ranks] = np.arange(nblocks)
    rep = first_idx[ranks]
    T2 = new_id[block[T[rep]]].astype(np.int32)
    return T2, out[rep].copy(), endout[rep].copy(), 0


def _byte_classes(d: Dfa) -> None:
    cols, inv = np.unique(d.trans, axis=1, return_inverse=True)
    d.cls = inv.reshape(-1).astype(np.uint8)
    d.ctrans = np.ascontiguousarray(cols)


# --------------------------------------------------------------------------- position automaton (bit-parallel NFA)
# For patterns whose DFA is too large (bounded gaps such as `a.{0,60}b` remember every recent start: the subset construction
# grows exponentially in the gap), the scan steps the NFA itself as a bit vector over its character edges ("positions",
# Glushkov form): every edge into position j consumes a code point of leaf(j), so one step is
#     D' = Follow(D, ctx) & B[class(c)]
#     Follow(D, ctx) = ((D << 1) & SHIFT) | (D & SELF) | OR_g [(D & SRC_g) != 0 and ctx in CTX_g] DST_g
# Assertions only read the code points on both sides of a boundary, so an epsilon path is valid under a set of
# (previous kind, next kind) context pairs: 5 kinds x 5 kinds = 25 bits.
K_EDGE, K_NL, K_WORD, K_UWORD, K_OTHER = range(5)     # start/end sentinel, '\n', \w in both senses, Unicode-only \w, other
N_KINDS = 5
CTX_ALL = (1 << (N_KINDS * N_KINDS)) - 1
PNA_MAX_POS = 256            # bits of the position vector, the virtual start bit included (8 words of 32)
PNA_MAX_CLASSES = 128
PNA_MAX_RANGES = 4096        # non-ASCII code point ranges (binary-searched in shared memory)
PNA_MAX_FOLLOW = 64
PNA_MAX_ACCEPT = 64
PNA_MAX_COUNTERS = 8         # counter positions (compile_positions_counted), each with its age in a register of the kernel


def ctx_bit(prev_kind: int, next_kind: int) -> int:
    return 1 << (prev_kind * N_KINDS + next_kind)


_PREV_CTX = {K_EDGE: (2, 0, 0), K_NL: (1, 0, 0), K_WORD: (0, 1, 1), K_UWORD: (0, 1, 0), K_OTHER: (0, 0, 0)}
_NEXT_CTX = {**_PREV_CTX, K_EDGE: (3, 0, 0)}


def _cond_ok(cond: int, prev, nxt) -> bool:
    """`cond_ok` of _determinize: prev / nxt are (nl: 0/1, 2 = start, 3 = end; uword; aword)."""
    if cond == A_BOS:
        return prev[0] == 2
    if cond == A_BOL:
        return prev[0] == 2 or prev[0] == 1
    if cond == A_EOS:
        return nxt[0] == 3
    if cond == A_EOL:
        return nxt[0] == 3 or nxt[0] == 1
    if cond == A_NEXTNL:
        return nxt[0] == 1
    if prev[0] == 2 and nxt[0] == 3:
        return False
    k = 1 if cond in (A_WB_U, A_NWB_U) else 2
    pw = prev[k] if prev[0] != 2 else 0
    nw = nxt[k] if nxt[0] != 3 else 0
    return (pw != nw) if cond in (A_WB_U, A_WB_A) else (pw == nw)


@dataclass
class Pna:
    """Position automaton of a pattern set.  Bit 0 is the virtual start position (set before the first character only);
    bit i >= 1 is character edge i of the NFA.  Masks are Python ints over n_pos bits."""
    n_words: int
    n_pos: int
    n_patterns: int
    ascii_cls: List[int]                      # [128] class of each ASCII code point
    ranges: List[Tuple[int, int]]             # sorted (first code point, class), covering 0x80 .. 0x10FFFF
    cls_b: List[int]                          # [class] positions whose leaf holds the class
    cls_kind: List[int]                       # [class] context kind
    shift: int
    self_loop: int
    start: int
    follow: List[Tuple[int, int, int]]        # (src, dst, ctx mask)
    accept: List[Tuple[int, int, int, bool]]  # (src, ctx mask, pattern, end only)
    counters: List[Tuple[int, int]] = field(default_factory=list)   # (position, bound k): position P holds `C{1,k}` (see run)

    def cls_of(self, cp: int) -> int:
        if cp < 0x80:
            return self.ascii_cls[cp]
        lo, hi = 0, len(self.ranges) - 1
        while lo < hi:
            mid = (lo + hi + 1) >> 1
            if self.ranges[mid][0] <= cp:
                lo = mid
            else:
                hi = mid - 1
        return self.ranges[lo][1]

    def follow_of(self, d: int, ctx: int) -> int:
        nd = ((d << 1) & self.shift) | (d & self.self_loop)
        for src, dst, m in self.follow:
            if m & ctx and d & src:
                nd |= dst
        return nd

    def accepts(self, d: int, ctx: int, at_end: bool) -> int:
        acc = 0
        for src, m, p, end_only in self.accept:
            if (at_end or not end_only) and m & ctx and d & src:
                acc |= 1 << p
        return acc

    def run(self, data: bytes) -> int:
        """Host simulation: mask of matching patterns for `data` (valid UTF-8), like Dfa.run.  A counter position P with bound k
        stays set while its class keeps matching and its age (code points since the newest entry) is below k:
            entered = F[P];  D'[P] = B[P] && (entered || (D[P] && age < k));  age = entered ? 1 : age + 1"""
        d, prev, acc = self.start, K_EDGE, 0
        age = [0] * len(self.counters)
        for ch in data.decode("utf-8", "surrogatepass"):
            c = self.cls_of(ord(ch))
            kind = self.cls_kind[c]
            ctx = ctx_bit(prev, kind)
            acc |= self.accepts(d, ctx, False)
            f = self.follow_of(d, ctx)
            nd = f
            for i, (p, k) in enumerate(self.counters):
                bit = 1 << p
                entered = f & bit
                if d & bit and age[i] < k:
                    nd |= bit
                age[i] = 1 if entered else age[i] + 1
            d = nd & self.cls_b[c]
            prev = kind
        return acc | self.accepts(d, ctx_bit(prev, K_EDGE), True)


def _positions(n: Nfa) -> List[Tuple[int, int, int]]:
    """Character edges (src, leaf, dst) reachable from the start, numbered depth-first with a state's character edges
    before its epsilon edges, so that a chain of characters gets consecutive numbers (follow edge i -> i + 1)."""
    out: List[Tuple[int, int, int]] = []
    seen = {n.start}
    stack = [(n.start, iter([("c", e) for e in n.chars[n.start]] + [("e", e) for e in n.eps[n.start]]))]
    while stack:
        s, it = stack[-1]
        nxt = next(it, None)
        if nxt is None:
            stack.pop()
            continue
        kind, e = nxt
        if kind == "c":
            leaf, d = e
            out.append((s, leaf, d))
        else:
            d = e[0]
        if d not in seen:
            seen.add(d)
            stack.append((d, iter([("c", x) for x in n.chars[d]] + [("e", x) for x in n.eps[d]])))
    return out


def compile_positions(patterns: Sequence[Pattern]) -> Pna:
    """Pattern set -> position automaton (pattern k = output bit k), from the same NFA compile_patterns determinizes."""
    if len(patterns) > 32:
        raise ValueError("at most 32 patterns per automaton")
    n = Nfa()
    for pid, p in enumerate(patterns):
        add_pattern(n, pid, p)
    n.add_trailing_newline_rule()
    return _pna_of(n, len(patterns))


def compile_positions_counted(patterns: Sequence[Pattern]) -> Pna:
    """compile_positions for pattern sets it refuses: countable repeats (`C{lo,hi}`, one character leaf C, finite hi) become
    lo expanded copies and one counter position each, the largest hi - lo first, until the automaton fits.  Within the
    repeat the expanded NFA holds one count per entry since C's current run began; all grow by one per character and the
    successors only need one in [1, k], so the newest entry's age is exact.  Raises PatternTooLarge when no number of
    counters (at most PNA_MAX_COUNTERS) makes it fit."""
    if len(patterns) > 32:
        raise ValueError("at most 32 patterns per automaton")
    cands = []                                        # (k, pattern, index into its _countable_repeats)
    for pid, p in enumerate(patterns):
        if p.kind == "regex":
            ast = _P.parse(p.text, p.flags)
            cands += [(k, pid, i) for i, (_node, k) in enumerate(_countable_repeats(ast.data, ast.state.flags, []))]
    cands.sort(key=lambda c: (-c[0], c[1], c[2]))
    why = "no repeat a counter can hold"
    for m in range(1, len(cands) + 1):
        chosen: Dict[int, List[int]] = {}
        for _k, pid, i in cands[:m]:
            chosen.setdefault(pid, []).append(i)
        n = Nfa()
        try:
            for pid, p in enumerate(patterns):
                add_pattern(n, pid, p, counted=chosen.get(pid, ()))
            n.add_trailing_newline_rule()
            return _pna_of(n, len(patterns))
        except PatternTooLarge as e:
            why = str(e)
    raise PatternTooLarge(f"position automaton with counters: {why}")


def _pna_of(n: Nfa, n_patterns: int) -> Pna:
    pos = _positions(n)
    n_pos = len(pos) + 1
    if n_pos > PNA_MAX_POS:
        raise PatternTooLarge(f"position automaton needs {n_pos} bits (limit {PNA_MAX_POS})")
    counters = [(i + 1, n.bound[e]) for i, e in enumerate(pos) if e in n.bound]
    if len(counters) > PNA_MAX_COUNTERS:
        raise PatternTooLarge(f"position automaton needs {len(counters)} counters (limit {PNA_MAX_COUNTERS})")
    counter_pos = {p for p, _k in counters}
    # code point classes: the leaves of the positions, plus the sets that decide a class' context kind
    uses = n.uses
    need_nl = A_BOL in uses or A_EOL in uses or A_NEXTNL in uses
    need_uw = bool(uses & {A_WB_U, A_NWB_U, A_WB_A, A_NWB_A})
    leaf_ids = sorted({leaf for _s, leaf, _d in pos})
    leaves = [n.leaves[x] for x in leaf_ids]
    ctx_leaf = {}
    if need_nl:
        ctx_leaf["nl"] = len(leaves); leaves.append(_NL)
    if need_uw:
        ctx_leaf["uw"] = len(leaves); leaves.append(_uword_set())
        ctx_leaf["aw"] = len(leaves); leaves.append(_AWORD)
    bounds, cls_of, members = _partition(leaves)
    ncls = len(members)
    if ncls > PNA_MAX_CLASSES:
        raise PatternTooLarge(f"position automaton needs {ncls} code point classes (limit {PNA_MAX_CLASSES})")

    def has(m, name):
        return name in ctx_leaf and (m >> ctx_leaf[name]) & 1

    kinds = [K_NL if has(m, "nl") else K_WORD if has(m, "aw") else K_UWORD if has(m, "uw") else K_OTHER for m in members]
    col = {leaf: k for k, leaf in enumerate(leaf_ids)}
    cls_b = [0] * ncls
    for i, (_s, leaf, _d) in enumerate(pos):
        bit = 1 << col[leaf]
        for c in range(ncls):
            if members[c] & bit:
                cls_b[c] |= 1 << (i + 1)
    ascii_cls = [int(cls_of[np.searchsorted(bounds, cp, side="right") - 1]) for cp in range(0x80)]
    ranges: List[Tuple[int, int]] = []
    for j in range(len(bounds) - 1):
        lo = int(bounds[j])
        if lo > MAX_CP:
            break
        lo = max(lo, 0x80)
        if int(bounds[j + 1]) <= lo:
            continue
        c = int(cls_of[j])
        if not ranges or ranges[-1][1] != c:
            ranges.append((lo, c))
    if len(ranges) > PNA_MAX_RANGES:
        raise PatternTooLarge(f"position automaton needs {len(ranges)} code point ranges (limit {PNA_MAX_RANGES})")

    # epsilon closures of every position's location under each of the 25 context pairs
    src_of: Dict[int, List[int]] = {}
    for i, (s, _leaf, _d) in enumerate(pos):
        src_of.setdefault(s, []).append(i + 1)
    locs = [n.start] + [d for _s, _leaf, d in pos]
    ctxs = [(pk, nk, ctx_bit(pk, nk), _PREV_CTX[pk], _NEXT_CTX[nk]) for pk in range(N_KINDS) for nk in range(N_KINDS)]
    shift = self_loop = 0
    follow: Dict[Tuple[int, int], int] = {}          # (dst set, ctx mask) -> src set
    accept: Dict[Tuple[int, int, bool], int] = {}    # (ctx mask, pattern, end only) -> src set
    for i, q in enumerate(locs):
        fm: Dict[int, int] = {}                      # position j -> ctx mask
        am: Dict[int, int] = {}                      # accepting state -> ctx mask
        for _pk, _nk, cb, pt, nt in ctxs:
            seen = {q}
            stack = [q]
            while stack:
                s = stack.pop()
                for dst, cond in n.eps[s]:
                    if dst not in seen and (cond == 0 or _cond_ok(cond, pt, nt)):
                        seen.add(dst); stack.append(dst)
            for s in seen:
                for j in src_of.get(s, ()):
                    fm[j] = fm.get(j, 0) | cb
                if s in n.accept:
                    am[s] = am.get(s, 0) | cb
        by_mask: Dict[int, int] = {}
        for j, m in fm.items():
            if m == CTX_ALL and j == i + 1:
                shift |= 1 << j
            elif m == CTX_ALL and j == i and j not in counter_pos:   # re-entering a counter is a fresh entry: a follow group
                self_loop |= 1 << j
            else:
                by_mask[m] = by_mask.get(m, 0) | (1 << j)
        for m, dst in by_mask.items():
            follow[(dst, m)] = follow.get((dst, m), 0) | (1 << i)
        for s, m in am.items():
            key = (m, n.accept[s], s in n.end_only)
            accept[key] = accept.get(key, 0) | (1 << i)
    if len(follow) > PNA_MAX_FOLLOW or len(accept) > PNA_MAX_ACCEPT:
        raise PatternTooLarge(f"position automaton needs {len(follow)} follow and {len(accept)} accept groups "
                              f"(limits {PNA_MAX_FOLLOW} / {PNA_MAX_ACCEPT})")
    words = 1
    while words * 32 < n_pos:
        words *= 2
    return Pna(n_words=words, n_pos=n_pos, n_patterns=n_patterns, ascii_cls=ascii_cls, ranges=ranges, cls_b=cls_b,
               cls_kind=kinds, shift=shift, self_loop=self_loop, start=1,
               follow=[(src, dst, m) for (dst, m), src in follow.items()],
               accept=[(src, m, p, eo) for (m, p, eo), src in accept.items()], counters=counters)
