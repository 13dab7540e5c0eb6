"""Position automata of head fields (header slots, flags, the five name fields) in the program blob: routing and bit
renumbering, the section layout (include/feiscan_prog.h fei_prog_slot.off_val_nfa, fei_prog_head_nfa), byte identity of
programs whose head fields all fit their DFAs, and every serialised head section read back through the CPU model
(tests/blob_nfa_model.py) against CPython re.search(p, value, re.I)."""
import hashlib
import random
import re
import struct

import pytest

import bench
from fei_b200 import program as P
from fei_b200.program import (C_BODY, C_DATE_CMP, C_FLAGS, C_NAME, C_SLOT, CMP, VERSION, VERSION_NFA, Cond, ProgramBuilder,
                              content_batch_program)
from fei_b200.regexc import Pattern, PatternTooLarge
from tests.blob_nfa_model import BlobNfa

# refused by the code-point DFA (subset construction over 30000 states), small as position automata
DEPLOY = r"deploy.{0,40}fail"                          # 2 words
URGENT = r"(urgent|asap).{0,30}(deploy|release)"       # 2 words
TICKET = r"[A-Z]{2,5}-\d{1,6}.{0,20}blocked"           # 2 words
SHORT = r"d.{0,16}f"                                   # 1 word


def _rx(p):
    return Pattern("regex", p, re.IGNORECASE)


def _program(queries):
    pb = ProgramBuilder()
    for q in queries:
        pb.add_query(q)
    return pb.build()


def _hdr(prog):
    v = struct.unpack_from("<24I", prog, 0)
    names = ("magic", "version", "total_bytes", "n_queries", "n_conds", "off_conds", "off_queries", "n_slots", "off_slots",
             "off_key_dfa", "off_body_dfa", "off_flags_dfa", "off_name0", "off_name1", "off_name2", "head_mask", "body_mask",
             "slot_mask", "name_mask", "head_bytes", "off_meta0", "off_meta1", "off_body_nfa", "off_head_nfa")
    return dict(zip(names, v))


def _slot(prog, k):
    return struct.unpack_from("<4I", prog, _hdr(prog)["off_slots"] + 16 * k)     # mode, off_val_dfa, empty_if_missing, off_val_nfa


def _head_nfa(prog):
    off = _hdr(prog)["off_head_nfa"]
    return struct.unpack_from("<6I", prog, off) if off else (0,) * 6              # flags, name fields 0..4


def _cond_bits(prog):
    h = _hdr(prog)
    return [struct.unpack_from("<4B", prog, h["off_conds"] + 32 * k) for k in range(h["n_conds"])]


def _dfa_patterns(prog, off):
    return struct.unpack_from("<I", prog, off + 36)[0] if off else 0             # fei_prog_dfa.n_outputs


def _check_section(prog, off, pats, first_bit, values):
    """The section at `off` holds `pats` as bits first_bit.. and agrees with re on every value."""
    m = BlobNfa(prog, off)
    assert (m.first_bit, m.n_patterns) == (first_bit, len(pats))
    end = m.table_bytes + struct.unpack_from("<I", prog, off + 32)[0]
    assert end <= _hdr(prog)["head_bytes"]                                        # staged with the program head
    for v in values:
        want = sum(1 << (first_bit + k) for k, p in enumerate(pats) if re.search(p, v, re.IGNORECASE))
        assert m.run(v.encode()) == want, (pats, v)


def _values(rng, n, pieces):
    return [""] + ["".join(rng.choice(pieces) for _ in range(rng.randint(0, 12))) for _ in range(n)]


PIECES = ["deploy", "DEPLOY", "fail", "urgent", "asap", "release", "ABC-123", "xy-1", "blocked", " ", "  ", "x" * 9, "é", "日本",
          "Σ", "σ", "ς", "İ", "i", "\n", "-", "d", "f", "k", "_", "ß", "K"]


def test_slot_with_one_proximity_pattern():
    prog = _program([[Cond(C_SLOT, pattern=_rx(DEPLOY), field="Subject")]])
    h = _hdr(prog)
    assert h["version"] == VERSION_NFA and h["off_body_nfa"] == 0 and h["off_head_nfa"] == 0
    mode, off_dfa, _empty, off_nfa = _slot(prog, 0)
    assert off_dfa == 0 and off_nfa                                               # the slot has only an automaton
    assert [b[2] for b in _cond_bits(prog)] == [0]
    assert BlobNfa(prog, off_nfa).W == 2
    _check_section(prog, off_nfa, [DEPLOY], 0, _values(random.Random(1), 200, PIECES))


def test_mixed_field_routes_and_renumbers():
    """Subject: a DFA pattern, a proximity one, another DFA one.  The DFA takes bits 0 and 1, the automaton bit 2."""
    subj = [_rx("urgent"), _rx(DEPLOY), _rx("asap|release")]
    queries = [[Cond(C_SLOT, pattern=subj[0], field="Subject")], [Cond(C_SLOT, pattern=subj[1], field="Subject", negate=True)],
               [Cond(C_SLOT, pattern=subj[2], field="Subject"), Cond(C_SLOT, pattern=subj[1], field="Subject")]]
    prog = _program(queries)
    _mode, off_dfa, _e, off_nfa = _slot(prog, 0)
    assert _dfa_patterns(prog, off_dfa) == 2 and off_nfa
    assert [(b[2], b[3]) for b in _cond_bits(prog)] == [(0, 0), (2, 1), (1, 0), (2, 0)]
    _check_section(prog, off_nfa, [DEPLOY], 2, _values(random.Random(2), 200, PIECES))


def test_refused_union_moves_the_largest(monkeypatch):
    """Every pattern fits the DFA alone but their union does not: the largest move to the automaton until the rest fits."""
    pats = [_rx("ab"), _rx(r"x.{0,5}y"), _rx("cd"), _rx(r"q.{0,7}z")]
    sizes = [P.cached_dfa([p]).n_states for p in pats]
    union = P.compile_patterns(pats).n_states
    limit = (max(sizes) + union) // 2
    assert max(sizes) < limit < union
    real = P.compile_patterns
    monkeypatch.setattr(P, "compile_patterns", lambda ps, sticky=False: real(ps, max_states=limit, sticky=sticky))
    monkeypatch.setattr(P, "_DFA_CACHE", {})
    monkeypatch.setattr(P, "_DFA_FAIL", {})
    dfa, nfa, a = P._route(pats, P._head_fits)
    assert nfa and a.n_patterns == len(nfa) and set(dfa) >= {0, 2}
    assert min(sizes[i] for i in nfa) >= max(sizes[i] for i in dfa)
    prog = _program([[Cond(C_SLOT, pattern=p, field="Subject")] for p in pats])
    _mode, off_dfa, _e, off_nfa = _slot(prog, 0)
    assert _dfa_patterns(prog, off_dfa) == len(dfa)
    order = [pats[i].text for i in dfa + nfa]
    assert [b[2] for b in _cond_bits(prog)] == [order.index(p.text) for p in pats]
    _check_section(prog, off_nfa, [pats[i].text for i in nfa], len(dfa), _values(random.Random(3), 200, ["ab", "x", "y", "q", "z", "--", "cd"]))


def test_head_and_body_automata_in_one_program():
    prog = _program([[Cond(C_SLOT, pattern=_rx(TICKET), field="Subject"), Cond(C_BODY, pattern=_rx(r"kubernetes.{0,60}docker"))],
                     [Cond(C_SLOT, pattern=_rx("python"), field="Tags")]])
    h = _hdr(prog)
    assert h["version"] == VERSION_NFA and h["off_body_nfa"] >= h["head_bytes"]      # the content automaton lies behind the head
    _mode, off_dfa, _e, off_nfa = _slot(prog, 0)
    assert off_dfa == 0 and off_nfa and _slot(prog, 1)[3] == 0
    _check_section(prog, off_nfa, [TICKET], 0, _values(random.Random(4), 200, PIECES))


def test_flags_and_name_fields():
    pats = {"flags": SHORT, 0: DEPLOY, 1: URGENT, 2: TICKET, 3: r"1.{0,20}7", 4: r"20.{0,40}:"}
    queries = [[Cond(C_FLAGS, pattern=_rx(pats["flags"]))]] + [[Cond(C_NAME, which=k, pattern=_rx(pats[k]))] for k in range(5)]
    prog = _program(queries)
    h = _hdr(prog)
    assert h["version"] == VERSION_NFA
    assert (h["off_flags_dfa"], h["off_name0"], h["off_name1"], h["off_name2"], h["off_meta0"], h["off_meta1"]) == (0,) * 6
    offs = _head_nfa(prog)
    assert all(offs) and h["off_head_nfa"] + 32 <= h["head_bytes"]
    rng = random.Random(5)
    _check_section(prog, offs[0], [pats["flags"]], 0, _values(rng, 200, ["D", "F", "S", "R", "P", "d", "f"]))
    digits = [str(d) for d in range(10)] + [" ", ":", "-", "20"]
    for k in range(5):
        _check_section(prog, offs[1 + k], [pats[k]], 0, _values(rng, 200, PIECES + digits))


def test_serialised_head_sections_agree_with_re():
    """Multi-byte UTF-8, word boundaries, anchors, (?m), empty values and the letters whose case folding differs between
    Unicode and ASCII (Σ σ ς, İ, K and the Kelvin sign)."""
    pats = [r"^deploy.{0,40}fail$", r"\bσ.{0,30}\bi", r"(?m)^d.{0,20}f$", r"İ.{0,30}k", r"\Bdeploy.{0,40}\bfail\b", r"ς.{0,40}ß$"]
    prog = _program([[Cond(C_SLOT, pattern=_rx(p), field="Subject", mode=2)] for p in pats])
    dfa, nfa, _a = P._route([_rx(p) for p in pats], P._head_fits)
    assert len(nfa) >= 4
    _mode, _off_dfa, _e, off_nfa = _slot(prog, 0)
    _check_section(prog, off_nfa, [pats[i] for i in nfa], len(dfa), _values(random.Random(6), 600, PIECES))


def test_limits_beyond_the_automaton_still_raise():
    with pytest.raises(PatternTooLarge):
        _program([[Cond(C_SLOT, pattern=_rx(r"a.{0,300}b"), field="Subject")]])       # more than 256 positions


def _fixed_programs():
    rx = _rx
    out = {"batch32": content_batch_program([rx(p) for p in bench.BATCH32])}
    from fei_b200.memdir_tools import filter as F
    pb = ProgramBuilder()
    for f in F.create_default_filters().filters:
        pb.add_query(F._compile_filter_conditions(f.conditions))
    out["default_filters"] = pb.build()
    out["cfg2"] = _program([[Cond(C_FLAGS, pattern=Pattern("exact_contains", "F")), Cond(C_DATE_CMP, op=CMP[">"], i64=1700000000 * 1000000),
                             Cond(C_SLOT, pattern=Pattern("has_tag", "python"), field="Tags", mode=0), Cond(C_BODY, pattern=rx(r"react|angular"))]])
    out["header_3_fields"] = _program([[Cond(C_SLOT, pattern=Pattern("has_tag", "python"), field="Tags", mode=0)],
                                       [Cond(C_SLOT, pattern=Pattern("contains", "learning"), field="Subject", mode=0)],
                                       [Cond(C_SLOT, pattern=Pattern("equals", "high"), field="Priority", mode=0),
                                        Cond(C_FLAGS, pattern=Pattern("exact_contains", "F"))]])
    out["body_nfa_only"] = content_batch_program([rx(r"kubernetes.{0,60}docker")])
    out["body_nfa_mixed"] = _program([[Cond(C_BODY, pattern=rx("python"))],
                                      [Cond(C_SLOT, pattern=Pattern("has_tag", "ta"), field="Tags"),
                                       Cond(C_BODY, pattern=rx(r"(error|fail).{0,80}(disk|memory)"))]])
    return out


# sha256 of the programs above as written before head fields had position automata
KNOWN = {
    "batch32": "c2dcc1e8801cf2244781eca9c6a897f20a3b00ecefac5de8125abe71a8881027",
    "default_filters": "0714d94413b079494665bafc4b6dcaa82cf1a3b46f83c84b25b34b8f185688ff",
    "cfg2": "ea219b569c74fbe4f36c447fd825d4e3c6c30181c7faf399f3667b2f40b8a1c5",
    "header_3_fields": "26fd73bfd0ca18e1841b006d3485b06ddf43527db28639ada675b8fd50aef3b0",
    "body_nfa_only": "b86a168c9123d251529ecbcc45d3c6141b07655e11939fda1871e3083006aaf4",
    "body_nfa_mixed": "3ff90de8038e7c49404d1fd7f307b702e167d6f8b351b14141b69009b96ad0f4",
}


def test_programs_whose_head_fields_fit_keep_their_bytes(monkeypatch):
    progs = _fixed_programs()
    assert {k: hashlib.sha256(v).hexdigest() for k, v in progs.items()} == KNOWN
    for k in ("batch32", "default_filters", "cfg2", "header_3_fields"):
        assert _hdr(progs[k])["version"] == VERSION and _hdr(progs[k])["off_head_nfa"] == 0, k
    # with the router forced to leave every head field to its DFA, nothing changes either
    route = P._route
    monkeypatch.setattr(P, "_route", lambda ps, fits, sticky=False: (list(range(len(ps))), [], None) if fits is P._head_fits
                        else route(ps, fits, sticky))
    assert _fixed_programs() == progs
