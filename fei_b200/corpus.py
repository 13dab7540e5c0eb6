"""Handle on a packed corpus resident in HBM (include/feiscan.h fei_corpus_*, fei_scan_*)."""
from __future__ import annotations

import ctypes as C
import os
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import _abi


class Corpus:
    """Pack once, scan many.  All compute goes through libfeiscan; there is no CPU path."""

    def __init__(self):
        _abi.init()
        self._h = C.c_void_p()
        _abi.check(_abi.lib().fei_corpus_create(C.byref(self._h)))
        self.n = 0
        self.global_base = 0

    def close(self) -> None:
        if self._h:
            _abi.lib().fei_corpus_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- filling
    def load(self, a: Dict[str, Any]) -> "Corpus":
        """`a`: canonical host arrays (fei_b200.synth.arrays_from_records / fei_b200.packer)."""
        h = _abi.CorpusHost()
        h.n = int(a["n"]); h.global_base = int(a.get("global_base", 0))
        for k in ("hdr", "hdr_off", "body", "body_off", "name", "name_off", "name_spans", "ts", "wall", "flags8", "fsb"):
            v = a.get(k)
            setattr(h, k, _abi.ptr(np.ascontiguousarray(v)) if v is not None else None)
        self._keep = a                      # arrays must outlive the call only, but keep them for materialisation
        _abi.check(_abi.lib().fei_corpus_load(self._h, C.byref(h)))
        self.n, self.global_base = h.n, h.global_base
        return self

    def load_raw(self, a: Dict[str, Any]) -> np.ndarray:
        """Raw ingest (fei_corpus_load_raw): `a` holds raw file bytes + meta columns.  Returns the validity flags;
        the corpus is loaded only when every file is valid UTF-8."""
        h = _abi.CorpusHost()
        h.n = int(a["n"]); h.global_base = int(a.get("global_base", 0))
        for k in ("name", "name_off", "name_spans", "ts", "wall", "flags8", "fsb"):
            v = a.get(k)
            setattr(h, k, _abi.ptr(np.ascontiguousarray(v)) if v is not None else None)
        valid = np.zeros(max(1, h.n), dtype=np.uint8)
        if "raw_begin" in a:                                            # files anywhere in the buffer; raw None = already staged on the device
            rc = _abi.lib().fei_corpus_load_raw_spans(self._h, C.byref(h), _abi.ptr(a["raw"]) if a["raw"] is not None else None, int(a["raw_bytes"]), _abi.ptr(a["raw_begin"]),
                                                      _abi.ptr(a["raw_len"]), _abi.ptr(valid))
        else:
            rc = _abi.lib().fei_corpus_load_raw(self._h, C.byref(h), _abi.ptr(a["raw"]), _abi.ptr(a["raw_off"]), _abi.ptr(valid))
        valid = valid[:h.n].astype(bool)
        if rc != 0 and not (_abi.lib().fei_last_error() or b"").startswith(b"some files are not valid UTF-8"):
            _abi.check(rc)                     # anything but "drop the undecodable files and load again" is an error
        if rc == 0:
            self._keep = None                  # every host array was consumed before the call returned (the text may be a transient arena)
            self.n, self.global_base = h.n, h.global_base
        return valid

    def stage_text(self, total: int, piece: np.ndarray, offset: int) -> None:
        """Uploads raw[offset : offset + len(piece)] of a text of `total` bytes ahead of load_raw (fei_corpus_stage_text)."""
        _abi.check(_abi.lib().fei_corpus_stage_text(self._h, int(total), piece.ctypes.data if len(piece) else None, int(offset), int(len(piece))))

    def fetch_meta(self) -> Dict[str, np.ndarray]:
        n = self.n
        ts = np.zeros(n, dtype=np.int64); wall = np.zeros(n, dtype=np.int64)
        f8 = np.zeros(n, dtype=np.uint64); fsb = np.zeros(n, dtype=np.uint32)
        _abi.check(_abi.lib().fei_corpus_fetch(self._h, 0, n, None, 0, None, None, 0, None, _abi.ptr(ts), _abi.ptr(wall), _abi.ptr(f8), _abi.ptr(fsb)))
        return {"ts": ts, "wall": wall, "flags8": f8, "fsb": fsb}

    def synth(self, seed: int, first: int, n: int) -> "Corpus":
        _abi.check(_abi.lib().fei_corpus_synth(self._h, seed, first, n))
        self.n, self.global_base = n, first
        return self

    def stats(self) -> Dict[str, int]:
        s = _abi.CorpusStats()
        _abi.check(_abi.lib().fei_corpus_stats_get(self._h, C.byref(s)))
        return {k: getattr(s, k) for k, _ in s._fields_}

    def fetch(self, first: int, n: int) -> Dict[str, Any]:
        """Canonical pieces of records [first, first+n) copied back from the device (bodies un-tiled)."""
        hdr_off = np.zeros(n + 1, dtype=np.uint64); body_off = np.zeros(n + 1, dtype=np.uint64)
        ts = np.zeros(n, dtype=np.int64); wall = np.zeros(n, dtype=np.int64)
        f8 = np.zeros(n, dtype=np.uint64); fsb = np.zeros(n, dtype=np.uint32)
        l = _abi.lib()
        _abi.check(l.fei_corpus_fetch(self._h, first, n, None, 0, _abi.ptr(hdr_off), None, 0, _abi.ptr(body_off),
                                      _abi.ptr(ts), _abi.ptr(wall), _abi.ptr(f8), _abi.ptr(fsb)))
        hdr = np.zeros(max(1, int(hdr_off[n])), dtype=np.uint8); body = np.zeros(max(1, int(body_off[n])), dtype=np.uint8)
        _abi.check(l.fei_corpus_fetch(self._h, first, n, _abi.ptr(hdr), hdr.size, None, _abi.ptr(body), body.size, None,
                                      None, None, None, None))
        return {"hdr": hdr, "hdr_off": hdr_off, "body": body, "body_off": body_off, "ts": ts, "wall": wall, "flags8": f8, "fsb": fsb}

    # ---- scanning
    def scan_masks(self, prog: bytes) -> np.ndarray:
        masks = np.zeros(max(1, self.n), dtype=np.uint32)
        _abi.check(_abi.lib().fei_scan_masks(self._h, prog, len(prog), _abi.ptr(masks)))
        return masks[:self.n]

    def scan_count(self, prog: bytes, nq: int) -> np.ndarray:
        counts = np.zeros(32, dtype=np.uint64)
        _abi.check(_abi.lib().fei_scan_count(self._h, prog, len(prog), _abi.ptr(counts)))
        return counts[:nq]

    def scan_hits(self, prog: bytes, nq: int, cap: Optional[int] = None) -> List[np.ndarray]:
        """Ordered global record indices per query."""
        if cap is None:                                  # one scan: counts first, then exactly-sized copies of the resident lists
            counts = self.scan_count(prog, nq)
            bufs = [np.empty(max(1, int(c)), dtype=np.uint64) for c in counts]
            ptrs = (C.c_void_p * 32)(*[_abi.ptr(b) for b in bufs])
            cap_arr = np.zeros(32, dtype=np.uint64); cap_arr[:nq] = counts
            _abi.check(_abi.lib().fei_scan_fetch_hits(self._h, nq, ptrs, _abi.ptr(cap_arr)))
            return [bufs[q][:int(counts[q])] for q in range(nq)]
        caps = [cap] * nq
        bufs = [np.zeros(max(1, c), dtype=np.uint64) for c in caps]
        ptrs = (C.c_void_p * 32)(*[_abi.ptr(b) for b in bufs])
        cap_arr = np.zeros(32, dtype=np.uint64); cap_arr[:nq] = caps
        nh = np.zeros(32, dtype=np.uint64)
        _abi.check(_abi.lib().fei_scan_hits(self._h, prog, len(prog), ptrs, _abi.ptr(cap_arr), _abi.ptr(nh)))
        return [bufs[q][:int(nh[q])] for q in range(nq)]

    def token_histogram(self, prog: bytes, sep: str = ",", cap: int = 32768, blob_cap: int = 1 << 22):
        """[(token bytes, count, global index of the first record carrying it)] in first-occurrence order
        (fei_corpus_token_histogram: the tag statistics of folders.py:286-292)."""
        blob = np.zeros(blob_cap, dtype=np.uint8); off = np.zeros(cap + 1, dtype=np.uint64)
        cnt = np.zeros(cap, dtype=np.uint64); first = np.zeros(cap, dtype=np.uint64)
        n = C.c_uint64()
        _abi.check(_abi.lib().fei_corpus_token_histogram(self._h, prog, len(prog), ord(sep), _abi.ptr(blob), blob_cap, _abi.ptr(off),
                                                         _abi.ptr(cnt), _abi.ptr(first), cap, C.byref(n)))
        raw = blob.tobytes()
        return [(raw[int(off[k]):int(off[k + 1])], int(cnt[k]), int(first[k])) for k in range(n.value)]

    def list_checksums(self, nq: int):
        """(A, S) per query of the ordered lists the last scan_count left on the device (fei_scan_list_checksum)."""
        a = np.zeros(32, dtype=np.uint64); s = np.zeros(32, dtype=np.uint64)
        _abi.check(_abi.lib().fei_scan_list_checksum(self._h, nq, _abi.ptr(a), _abi.ptr(s)))
        return a[:nq], s[:nq]

    def fetch_records(self, idx: np.ndarray, want_body: bool = True):
        """Header text and body of arbitrary records (fei_corpus_fetch_records): (hdr bytes, hdr_off[m+1], body bytes, body_off[m+1])."""
        idx = np.ascontiguousarray(idx, dtype=np.uint64)
        m = idx.size
        ho = np.zeros(m + 1, dtype=np.uint64); bo = np.zeros(m + 1, dtype=np.uint64)
        l = _abi.lib()
        _abi.check(l.fei_corpus_fetch_records(self._h, _abi.ptr(idx), m, None, 0, _abi.ptr(ho), None, 0, _abi.ptr(bo)))
        hdr = np.zeros(max(1, int(ho[m])), dtype=np.uint8)
        body = np.zeros(max(1, int(bo[m])) if want_body else 1, dtype=np.uint8)
        _abi.check(l.fei_corpus_fetch_records(self._h, _abi.ptr(idx), m, _abi.ptr(hdr), hdr.size, _abi.ptr(ho),
                                              _abi.ptr(body) if want_body else None, body.size, _abi.ptr(bo)))
        return hdr[:int(ho[m])].tobytes(), ho, (body[:int(bo[m])].tobytes() if want_body else b""), bo

    def save(self, path: str) -> None:
        _abi.check(_abi.lib().fei_corpus_save(self._h, os.fsencode(path)))

    def load_snapshot(self, path: str) -> float:
        """Restores a corpus saved with save(); returns the restore rate in GB/s (CUDA events around the upload)."""
        gbs = C.c_float()
        _abi.check(_abi.lib().fei_corpus_load_snapshot(self._h, os.fsencode(path), C.byref(gbs)))
        st = self.stats()
        self.n, self.global_base = st["n"], st["global_base"]
        return float(gbs.value)

    def slot_values(self, prog: bytes):
        """The header value the reference would read for slot 0 of `prog`, record by record (fei_corpus_slot_values):
        (present[n] bool, off[n+1], blob bytes)."""
        n = self.n
        present = np.zeros(max(1, n), dtype=np.uint8); off = np.zeros(n + 1, dtype=np.uint64)
        blob = np.zeros(max(64, 24 * n), dtype=np.uint8)
        l = _abi.lib()
        rc = l.fei_corpus_slot_values(self._h, prog, len(prog), _abi.ptr(present), _abi.ptr(off), _abi.ptr(blob), blob.size)
        if rc == _abi.FEI_E_CAPACITY:
            blob = np.zeros(int(off[n]) + 16, dtype=np.uint8)
            rc = l.fei_corpus_slot_values(self._h, prog, len(prog), _abi.ptr(present), _abi.ptr(off), _abi.ptr(blob), blob.size)
        _abi.check(rc)
        return present[:n].astype(bool), off, blob[:int(off[n])]

    TAG_OPS = {"add": 0, "remove": 1, "replace": 2}

    def tag_edit(self, prog: bytes, operation: str, tags: Sequence[bytes]):
        """The records of `prog`'s query whose `Tags` multiset `operation` changes (fei_corpus_tag_edit: the tag edit of
        folders.py:483-587; header field 0 of `prog` is the exact key Tags, field 1 the exact key Subject).  Returns
        (global indices, [(Subject bytes or None, old tags bytes, new tags bytes)]) in corpus order."""
        blob = b"".join(tags)
        toff = np.zeros(len(tags) + 1, dtype=np.uint64)
        toff[1:] = np.cumsum([len(t) for t in tags], dtype=np.uint64)
        src = np.frombuffer(blob, dtype=np.uint8) if blob else np.zeros(1, dtype=np.uint8)
        l = _abi.lib()
        cap, text_cap = max(1, self.n), 64 * max(1, self.n)       # an exact retry below when the text does not fit
        while True:
            rec = np.empty(cap, dtype=np.uint64); text = np.empty(text_cap, dtype=np.uint8)
            off = np.empty(3 * cap + 1, dtype=np.uint64); has = np.empty(cap, dtype=np.uint8)
            m = C.c_uint64()
            rc = l.fei_corpus_tag_edit(self._h, prog, len(prog), self.TAG_OPS[operation], _abi.ptr(src), _abi.ptr(toff), len(tags),
                                       _abi.ptr(rec), cap, C.byref(m), _abi.ptr(text), text_cap, _abi.ptr(off), _abi.ptr(has))
            if rc != _abi.FEI_E_CAPACITY:
                break
            cap, text_cap = max(1, m.value), max(1, int(off[0]))
        _abi.check(rc)
        k = m.value
        raw = text[:int(off[3 * k])].tobytes()
        o = off[:3 * k + 1].tolist()
        out = [(raw[o[3 * j]:o[3 * j + 1]] if has[j] else None, raw[o[3 * j + 1]:o[3 * j + 2]], raw[o[3 * j + 2]:o[3 * j + 3]]) for j in range(k)]
        return rec[:k].copy(), out

    def format_records(self, idx: np.ndarray, fmt: int, opts: int, folder_names: Sequence[bytes], cap: Optional[int] = None):
        """What the command line prints for records idx (corpus-local, output order), written on the GPU (fei_corpus_format_records,
        formats _abi.FEI_FMT_*): (bytes, offsets[m+1]).  With `cap`, at most that many bytes: when the records need more, returns
        (None, offsets) so the caller can take a prefix that fits."""
        idx = np.ascontiguousarray(idx, dtype=np.uint64)
        m = idx.size
        names = b"".join(folder_names)
        fblob = np.frombuffer(names, dtype=np.uint8) if names else np.zeros(1, dtype=np.uint8)
        foff = np.zeros(len(folder_names) + 1, dtype=np.uint64)
        foff[1:] = np.cumsum([len(f) for f in folder_names], dtype=np.uint64)
        off = np.zeros(m + 1, dtype=np.uint64)
        l = _abi.lib()
        ms = C.c_float()
        size = cap if cap is not None else 0
        while True:
            out = np.empty(max(1, size), dtype=np.uint8)
            rc = l.fei_corpus_format_records(self._h, _abi.ptr(idx), m, fmt, opts, _abi.ptr(fblob), _abi.ptr(foff), len(folder_names),
                                             _abi.ptr(out), size, _abi.ptr(off), C.byref(ms))
            if rc != _abi.FEI_E_CAPACITY or cap is not None:
                break
            size = int(off[m])                                      # sized by the failed call: the retry fits
        self.last_format_ms = float(ms.value)
        if rc == _abi.FEI_E_CAPACITY:
            return None, off
        _abi.check(rc)
        return out[:int(off[m])].tobytes(), off

    def set_aux(self, k: int, verdicts: Optional[np.ndarray]) -> None:
        """Aux column k: one host-computed verdict byte per record, read by C_RECBITS conditions (fei_corpus_set_aux)."""
        if verdicts is None:
            _abi.check(_abi.lib().fei_corpus_set_aux(self._h, k, None, 0))
            return
        v = np.ascontiguousarray(verdicts, dtype=np.uint8)
        _abi.check(_abi.lib().fei_corpus_set_aux(self._h, k, _abi.ptr(v), v.size))

    def timing(self) -> Dict[str, float]:
        t = _abi.ScanTiming()
        _abi.check(_abi.lib().fei_scan_last_timing(self._h, C.byref(t)))
        return {k: getattr(t, k) for k, _ in t._fields_}

    @property
    def handle(self):
        return self._h
