"""Memorychain link-hash validation on the GPU.

Mirror of the hot part of the reference's ``memdir_tools/memorychain.py``:

* ``MemoryBlock``            — fields, ``calculate_hash``, ``to_dict`` / ``from_dict``
  (reference :74-130, :263-327)
* ``MemoryChain.validate_chain`` — same signature and log lines (reference :596-618)
* ``validate_chain_blocks``  — the drop-in body for the reference's own class: works on
  any sequence of objects exposing the reference's block attributes.

All hashing goes through ``libfeiscan.so`` (``fei_chain_validate_cols``): the host only
marshals the ten hashed fields into typed columns; canonical JSON is produced by the
library's C++ serialiser and SHA-256 + the two comparisons run in the CUDA kernel
(``fei_b200/csrc/chain.cu``).  There is no hashlib path.
"""
from __future__ import annotations

import ctypes as C
import json
import logging
import os
import threading
import weakref
import time
from operator import attrgetter, itemgetter
from typing import Any, Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np

from .. import _abi

try:                                    # CPython helper built by `make` (fei_b200/_fastcols.c); host glue only: without it the
    from .. import _fastcols            # pure-Python marshalling below does the same job, slower
except ImportError:                     # pragma: no cover
    _fastcols = None

logger = logging.getLogger("memorychain")     # same logger name as the reference (:43)

CHAIN_FILE = os.path.join(os.path.expanduser("~"), ".memdir", "memorychain.json")     # reference :49

TASK_PROPOSED = "proposed"
DIFFICULTY_LEVELS = {"easy": 1, "medium": 3, "hard": 5, "very_hard": 10, "extreme": 20}

# sorted key order of the hashed dict (reference :117-128 with sort_keys=True)
HASHED_FIELDS = ("difficulty", "index", "memory_id", "nonce", "previous_hash",
                 "proposer_node", "responsible_node", "solver_node", "task_state", "timestamp")


# --------------------------------------------------------------------------- marshalling
class _Col:
    """One typed JSON column (include/feiscan.h fei_json_col) with its backing arrays."""

    __slots__ = ("tag", "uniform", "num", "blob", "off")

    def __init__(self):
        self.tag = None; self.uniform = _abi.J_NULL; self.num = None; self.blob = None; self.off = None

    def fill(self, dst: _abi.JsonCol) -> None:
        dst.tag = _abi.ptr(self.tag)
        dst.uniform_tag = self.uniform
        dst.num = _abi.ptr(self.num)
        dst.str = _abi.ptr(self.blob)
        dst.str_off = _abi.ptr(self.off)


def _str_blob(vals: Sequence[str]) -> Tuple[np.ndarray, np.ndarray]:
    n = len(vals)
    lens = np.fromiter(map(len, vals), dtype=np.int64, count=n)
    blob = "".join(vals).encode("utf-8", "surrogatepass")
    if len(blob) != int(lens.sum()):       # non-ASCII somewhere: byte lengths differ from str lengths
        enc = [v.encode("utf-8", "surrogatepass") for v in vals]
        lens = np.fromiter(map(len, enc), dtype=np.int64, count=n)
        blob = b"".join(enc)
    off = np.zeros(n + 1, dtype=np.uint64)
    np.cumsum(lens, out=off[1:])
    arr = np.frombuffer(blob, dtype=np.uint8) if blob else np.zeros(1, dtype=np.uint8)
    return arr, off


def _column(vals: Sequence[Any], what: str) -> _Col:
    """Typed column for values json.dumps would emit as scalars."""
    col = _Col()
    n = len(vals)
    kinds = set(map(type, vals))
    if kinds == {str}:
        col.uniform = _abi.J_STR
        col.blob, col.off = _str_blob(vals)
        return col
    if kinds == {float}:
        col.uniform = _abi.J_FLOAT
        col.num = np.array(vals, dtype=np.float64).view(np.uint64)
        return col
    if kinds == {int}:
        try:
            col.num = np.array(vals, dtype=np.int64).view(np.uint64)
            col.uniform = _abi.J_INT
            return col
        except OverflowError:
            pass
    if kinds == {type(None)}:
        col.uniform = _abi.J_NULL
        return col
    # mixed / exotic: per-element tags
    tag = np.zeros(n, dtype=np.uint8)
    num = np.zeros(n, dtype=np.uint64)
    strs: List[str] = [""] * n
    for i, v in enumerate(vals):
        if v is None:
            tag[i] = _abi.J_NULL
        elif v is True:
            tag[i] = _abi.J_TRUE
        elif v is False:
            tag[i] = _abi.J_FALSE
        elif isinstance(v, str):
            tag[i] = _abi.J_STR; strs[i] = str.__str__(v)
        elif isinstance(v, int):
            iv = int(v)
            if -(1 << 63) <= iv < (1 << 63):
                tag[i] = _abi.J_INT; num[i] = np.int64(iv).view(np.uint64)
            else:
                tag[i] = _abi.J_BIGINT; strs[i] = int.__repr__(iv)
        elif isinstance(v, float):
            tag[i] = _abi.J_FLOAT; num[i] = np.float64(v).view(np.uint64)
        else:
            raise NotImplementedError(
                f"block field {what!r} holds a {type(v).__name__}; only JSON scalars are hashed on the GPU")
    col.tag, col.num = tag, num
    col.blob, col.off = _str_blob(strs)
    return col


_get_direct = attrgetter("index", "nonce", "previous_hash", "proposer_node", "responsible_node", "timestamp", "memory_data", "hash")


_EMPTY: Dict[str, Any] = {}


def _memory_id(md: Any) -> Any:
    # self.memory_data.get("metadata", {}).get("unique_id", "")   (reference :120)
    return md.get("metadata", {}).get("unique_id", "")


_DIRECT = ("index", "nonce", "previous_hash", "proposer_node", "responsible_node", "timestamp", "memory_data")
_OPTIONAL = ("task_state", "difficulty", "solver_node")
_get_dict = attrgetter("__dict__")


def _plain_hash_key(blocks: Sequence[Any]) -> Optional[str]:
    """The instance-dict key of the stored hash when every block is a plain instance of one class whose hashed fields are
    ordinary instance attributes, else None: the one test both fast column paths (_extract, chain_columns_native) share."""
    kinds = set(map(type, blocks))
    if len(kinds) != 1:
        return None
    cls = kinds.pop()
    hash_key = "hash"
    if isinstance(getattr(cls, "hash", None), property):
        if cls is not MemoryBlock and cls is not _TrackedBlock:
            return None
        hash_key = "_hash"                       # our lazy-hash block keeps the value there (None until first use)
    elif hasattr(cls, "hash"):
        return None
    if any(hasattr(cls, k) for k in _DIRECT + _OPTIONAL) or hasattr(cls, "__getattr__"):
        return None                              # class-level attributes / descriptors / dynamic lookup: use getattr
    return hash_key


def _extract(blocks: Sequence[Any]) -> Optional[List[tuple]]:
    """Fast attribute extraction: when the blocks are plain (_plain_hash_key), read the hashed fields straight out of the
    instance dicts (C speed, no descriptor protocol).
    Returns 11 tuples (7 direct, hash, 3 optional) or None when the generic getattr path must be used."""
    hash_key = _plain_hash_key(blocks)
    if hash_key is None:
        return None
    try:
        rows = list(map(itemgetter(*_DIRECT, hash_key, *_OPTIONAL), map(_get_dict, blocks)))
    except (AttributeError, KeyError):           # __slots__ classes, blocks without task fields (getattr(..., None))
        return None
    cols = list(zip(*rows))
    if hash_key == "_hash" and None in cols[7]:
        cols[7] = tuple(b.hash if h is None else h for b, h in zip(blocks, cols[7]))
    return cols


def _col_from_native(t: tuple) -> _Col:
    col = _Col()
    kind = t[0]
    if kind == 1:
        col.uniform = _abi.J_STR
        col.blob = np.frombuffer(t[1], dtype=np.uint8) if t[1] else np.zeros(1, dtype=np.uint8)
        col.off = np.frombuffer(t[2], dtype=np.uint64)
    elif kind == 2:
        col.uniform = _abi.J_INT; col.num = np.frombuffer(t[1], dtype=np.uint64)
    elif kind == 3:
        col.uniform = _abi.J_FLOAT; col.num = np.frombuffer(t[1], dtype=np.uint64)
    else:
        col.uniform = _abi.J_NULL
    return col


_NATIVE_NAMES = {"memory_id": "memory_data"}          # hashed field -> instance attribute it is read from


def chain_columns_native(blocks: Sequence[Any]) -> Optional[Tuple[List[_Col], np.ndarray, np.ndarray]]:
    """The ten hashed columns + the stored-hash blob through the C helper, or None when the blocks are not plain enough
    for it (then chain_columns decides)."""
    if _fastcols is None or not blocks:
        return None
    hash_key = _plain_hash_key(blocks)
    if hash_key is None:
        return None
    names = tuple(_NATIVE_NAMES.get(k, k) for k in HASHED_FIELDS) + (hash_key,)
    out = _fastcols.columns(blocks if isinstance(blocks, list) else list(blocks), names, HASHED_FIELDS.index("memory_id"))
    if out is None or out[-1][0] != 1:                  # unusual values somewhere / hashes not (all) strings yet
        return None
    cols = [_col_from_native(t) for t in out[:-1]]
    h = out[-1]
    return cols, (np.frombuffer(h[1], dtype=np.uint8) if h[1] else np.zeros(1, dtype=np.uint8)), np.frombuffer(h[2], dtype=np.uint64)


def chain_columns(blocks: Sequence[Any]) -> Tuple[List[_Col], List[Any]]:
    """Ten hashed columns (sorted key order) + the stored ``hash`` attributes."""
    fast = _extract(blocks) if blocks else None
    if fast is not None:
        index, nonce, prev, proposer, responsible, timestamp, mdata, stored, task_state, difficulty, solver = fast
    else:
        rows = list(map(_get_direct, blocks))
        if rows:
            index, nonce, prev, proposer, responsible, timestamp, mdata, stored = map(list, zip(*rows))
        else:
            index = nonce = prev = proposer = responsible = timestamp = mdata = stored = []
        # getattr(self, "task_state", None) etc. (reference :124-126)
        task_state = [getattr(b, "task_state", None) for b in blocks]
        difficulty = [getattr(b, "difficulty", None) for b in blocks]
        solver = [getattr(b, "solver_node", None) for b in blocks]
    try:                                         # self.memory_data.get("metadata", {}).get("unique_id", "")   (reference :120)
        memory_id = [md.get("metadata", _EMPTY).get("unique_id", "") for md in mdata]
    except AttributeError:
        memory_id = list(map(_memory_id, mdata))
    by_name = {"difficulty": difficulty, "index": index, "memory_id": memory_id, "nonce": nonce,
               "previous_hash": prev, "proposer_node": proposer, "responsible_node": responsible,
               "solver_node": solver, "task_state": task_state, "timestamp": timestamp}
    return [_column(by_name[k], k) for k in HASHED_FIELDS], stored


def _cols_struct(cols: List[_Col]):
    arr = (_abi.JsonCol * _abi.CHAIN_NCOLS)()
    for k, c in enumerate(cols):
        c.fill(arr[k])
    return arr


def canonical_texts(blocks: Sequence[Any]) -> List[bytes]:
    """The exact byte strings the reference feeds to sha256 (host serialiser only; used by tests)."""
    cols, _ = chain_columns(blocks)
    n = len(blocks)
    off = np.zeros(n + 1, dtype=np.uint64)
    cap = max(1024, 1024 * n)
    buf = np.zeros(cap, dtype=np.uint8)
    arr = _cols_struct(cols)
    _abi.check(_abi.lib().fei_chain_serialize_cols(arr, n, _abi.ptr(buf), cap, _abi.ptr(off)))
    return [bytes(buf[int(off[i]):int(off[i + 1])]) for i in range(n)]


def hash_and_validate(blocks: Sequence[Any], first_index: int = 0, want_digests: bool = False
                      ) -> Tuple[int, int, Optional[np.ndarray]]:
    """GPU pass over ``blocks``: returns (first_bad or -1, kind, digests[n,32] or None).

    kind 1 = "invalid hash", 2 = "broken link to previous block"; element 0 is only used
    as a predecessor (the reference never checks the genesis block, :604).
    """
    _abi.init()
    n = len(blocks)
    native = chain_columns_native(blocks)
    if native is not None:
        cols, hash_blob, hash_off = native
    else:
        cols, stored = chain_columns(blocks)
        if not all(isinstance(h, str) for h in stored):
            # `!=` between arbitrary objects (None == None ...) has no string form
            raise NotImplementedError("block.hash must be a str for GPU validation")
        hash_blob, hash_off = _str_blob(stored)
    first_bad, kind = C.c_int64(-1), C.c_int32(0)
    digests = np.zeros((n, 32), dtype=np.uint8) if want_digests else None
    arr = _cols_struct(cols)
    _abi.check(_abi.lib().fei_chain_validate_cols(
        arr, _abi.ptr(hash_blob), _abi.ptr(hash_off), n, first_index,
        C.byref(first_bad), C.byref(kind), _abi.ptr(digests), None, 0, None))
    return first_bad.value, kind.value, digests


def validate_chain_blocks(chain: Sequence[Any], lock: Optional[Any] = None, log: logging.Logger = logger) -> bool:
    """Drop-in body of ``MemoryChain.validate_chain`` (reference :596-618)."""
    ctx = lock if lock is not None else threading.RLock()
    with ctx:
        if len(chain) < 2:
            return True
        first_bad, kind, _ = hash_and_validate(chain)
    if first_bad < 0:
        return True
    if kind == 1:
        log.error(f"Block {first_bad} has invalid hash")
    else:
        log.error(f"Block {first_bad} has broken link to previous block")
    return False


# --------------------------------------------------------------------------- reference-shaped classes
class MemoryBlock:
    """Same constructor, attributes and (de)serialisation as the reference block (:74-108, :263-327).

    ``hash`` is computed lazily on first access (the reference hashes eagerly in the
    constructor and again after ``from_dict`` overwrites it); the value is identical.
    """

    def __init__(self, index: int, timestamp: float, memory_data: Dict[str, Any],
                 previous_hash: str, responsible_node: str, proposer_node: str):
        self.index = index
        self.timestamp = timestamp
        self.memory_data = memory_data
        self.previous_hash = previous_hash
        self.responsible_node = responsible_node
        self.proposer_node = proposer_node
        self.nonce = 0
        self.working_nodes: List[str] = []
        self.solutions: List[Any] = []
        self.difficulty = memory_data.get("task_difficulty", "medium")
        self.reward = DIFFICULTY_LEVELS.get(self.difficulty, 3)
        self.task_state = memory_data.get("task_state", TASK_PROPOSED)
        self.solver_node = None
        self.difficulty_votes: Dict[str, Any] = {}
        self._hash: Optional[str] = None

    @property
    def hash(self) -> str:
        if self._hash is None:
            self._hash = self.calculate_hash()
        return self._hash

    @hash.setter
    def hash(self, value: str) -> None:
        self._hash = value

    def calculate_hash(self) -> str:
        probe = _HashProbe(self)
        _, _, dig = hash_and_validate([probe], want_digests=True)
        return bytes(dig[0]).hex()

    def mine_block(self, difficulty: int = 2, max_tries: int = 1 << 40) -> None:
        """Proof of work on the GPU (reference :132-143): smallest nonce >= the current one whose hash starts with
        `difficulty` zeros.  The canonical text only differs in the nonce digits, so the host serialises it twice
        (nonce 0 and 1) to cut prefix / suffix and the kernel tries one candidate nonce per thread."""
        if not isinstance(self.nonce, int) or isinstance(self.nonce, bool) or self.nonce < 0:
            raise NotImplementedError("mine_block needs a non-negative int nonce")
        keep = self.nonce
        try:
            self.nonce = 0
            t0 = canonical_texts([_HashProbe(self)])[0]
            self.nonce = 1
            t1 = canonical_texts([_HashProbe(self)])[0]
        finally:
            self.nonce = keep
        pos = next(i for i in range(len(t0)) if t0[i] != t1[i])
        prefix, suffix = t0[:pos], t0[pos + 1:]
        _abi.init()
        nonce, tried = C.c_uint64(), C.c_uint64()
        digest = np.zeros(32, dtype=np.uint8)
        _abi.check(_abi.lib().fei_chain_mine(prefix, len(prefix), suffix, len(suffix), keep, int(difficulty), int(max_tries),
                                             C.byref(nonce), _abi.ptr(digest), C.byref(tried)))
        self.nonce = int(nonce.value)
        self.hash = bytes(digest).hex()

    def is_task(self) -> bool:
        return self.memory_data.get("type") == "task"

    def to_dict(self) -> Dict[str, Any]:
        data = {"index": self.index, "timestamp": self.timestamp, "memory_data": self.memory_data,
                "previous_hash": self.previous_hash, "responsible_node": self.responsible_node,
                "proposer_node": self.proposer_node, "nonce": self.nonce, "hash": self.hash}
        if self.is_task():
            data.update({"working_nodes": self.working_nodes, "solutions": self.solutions,
                         "difficulty": self.difficulty, "reward": self.reward, "task_state": self.task_state,
                         "solver_node": self.solver_node, "difficulty_votes": self.difficulty_votes})
        return data

    @classmethod
    def from_dict(cls, data: Dict[str, Any]) -> "MemoryBlock":
        block = cls(data["index"], data["timestamp"], data["memory_data"], data["previous_hash"],
                    data["responsible_node"], data["proposer_node"])
        block.nonce = data["nonce"]
        block.hash = data["hash"]
        if block.is_task():
            block.working_nodes = data.get("working_nodes", [])
            block.solutions = data.get("solutions", [])
            block.difficulty = data.get("difficulty", "medium")
            block.reward = data.get("reward", DIFFICULTY_LEVELS.get(block.difficulty, 3))
            block.task_state = data.get("task_state", TASK_PROPOSED)
            block.solver_node = data.get("solver_node")
            block.difficulty_votes = data.get("difficulty_votes", {})
        return block


class _HashProbe:
    """View of a block whose stored hash is irrelevant (single-block hashing)."""
    hash = ""

    def __init__(self, b: Any):
        self.__dict__.update({k: getattr(b, k) for k in
                              ("index", "nonce", "previous_hash", "proposer_node", "responsible_node",
                               "timestamp", "memory_data")})
        for k in ("task_state", "difficulty", "solver_node"):
            if hasattr(b, k):
                setattr(self, k, getattr(b, k))



# --------------------------------------------------------------------------- resident chain
_WATCHED = frozenset(_DIRECT + _OPTIONAL + ("hash", "_hash"))


class _TrackedBlock(MemoryBlock):
    """A MemoryBlock that sits in a MemoryChain: assigning one of its hashed attributes (or its stored hash) tells the chain that
    its device image is stale from that block on.  Blocks are switched to this class when they enter a chain (same layout), so
    building blocks stays as cheap as a plain class."""

    def __setattr__(self, name, value):
        object.__setattr__(self, name, value)
        if name in _WATCHED:
            for ref, pos in self.__dict__.get("_fei_owners", ()):
                chain = ref()
                if chain is not None:
                    chain._touch(pos)


def _track(block: Any, chain: "MemoryChain", pos: int) -> None:
    if type(block) is MemoryBlock:
        object.__setattr__(block, "__class__", _TrackedBlock)
    if type(block) is _TrackedBlock:
        owners = [(r, p) for r, p in block.__dict__.get("_fei_owners", ()) if r() is not None and r() is not chain]
        owners.append((weakref.ref(chain), pos))
        block.__dict__["_fei_owners"] = owners


class _TrackedList(list):
    """`MemoryChain.chain`: a list whose structural changes (append, item assignment, insert, delete, sort ...) mark the chain's
    device image stale from the lowest index they can affect."""

    def __init__(self, owner: "MemoryChain", items=()):
        super().__init__(items)
        self._owner = weakref.ref(owner)

    def _dirty(self, k: int) -> None:
        o = self._owner()
        if o is not None:
            o._touch(max(0, k))

    def append(self, x): self._dirty(len(self)); super().append(x)
    def extend(self, xs): self._dirty(len(self)); super().extend(xs)
    def insert(self, i, x): self._dirty(i if i >= 0 else len(self) + i); super().insert(i, x)
    def pop(self, i=-1): self._dirty(i if i >= 0 else len(self) + i); return super().pop(i)
    def remove(self, x): self._dirty(0); super().remove(x)
    def clear(self): self._dirty(0); super().clear()
    def sort(self, *a, **k): self._dirty(0); super().sort(*a, **k)
    def reverse(self): self._dirty(0); super().reverse()
    def __iadd__(self, xs): self._dirty(len(self)); return super().__iadd__(xs)
    def __imul__(self, k): self._dirty(0); return super().__imul__(k)

    def __setitem__(self, i, x):
        self._dirty(0 if isinstance(i, slice) else (i if i >= 0 else len(self) + i))
        super().__setitem__(i, x)

    def __delitem__(self, i):
        self._dirty(0 if isinstance(i, slice) else (i if i >= 0 else len(self) + i))
        super().__delitem__(i)


class _Resident:
    """Device image of a chain (fei_chain*): the hashed fields as typed columns, turned into canonical JSON and SHA-ready blocks
    by GPU kernels once (fei_chain_load_cols); every validate_chain() after that re-hashes what is resident (fei_chain_validate)."""

    def __init__(self):
        _abi.init()
        self.h = C.c_void_p()
        _abi.check(_abi.lib().fei_chain_create(C.byref(self.h)))
        self.n = 0
        self.cols: Optional[List[_Col]] = None           # host copy of the columns: a changed tail is re-marshalled, the rest reused
        self.hash_blob: Optional[np.ndarray] = None
        self.hash_off: Optional[np.ndarray] = None
        self.uploads = 0
        self.marshalled = 0

    def close(self) -> None:
        if self.h:
            _abi.lib().fei_chain_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _marshal(blocks: Sequence[Any]):
        native = chain_columns_native(blocks)
        if native is not None:
            return native
        cols, stored = chain_columns(blocks)
        if not all(isinstance(h, str) for h in stored):
            raise NotImplementedError("block.hash must be a str for GPU validation")
        hb, ho = _str_blob(stored)
        return cols, hb, ho

    @staticmethod
    def _concat(a: _Col, b: _Col, na: int) -> Optional[_Col]:
        """Column a (first na entries) followed by column b; None when their representations differ (then everything is re-marshalled)."""
        if a.tag is not None or b.tag is not None or a.uniform != b.uniform:
            return None
        c = _Col()
        c.uniform = a.uniform
        if a.uniform in (_abi.J_INT, _abi.J_FLOAT):
            c.num = np.concatenate([a.num[:na], b.num])
        elif a.uniform == _abi.J_STR:
            end = int(a.off[na])
            c.blob = np.concatenate([a.blob[:end], b.blob]) if end or len(b.blob) else np.zeros(1, dtype=np.uint8)
            c.off = np.concatenate([a.off[:na + 1], b.off[1:] + np.uint64(end)])
        return c

    def sync(self, blocks: Sequence[Any], dirty_from: Optional[int]) -> bool:
        """Bring the device image in line with `blocks`; False when this chain cannot be resident (falls back to one-shot calls)."""
        n = len(blocks)
        keep = 0
        if self.cols is not None and dirty_from is not None:
            keep = min(dirty_from, self.n, n)
        elif self.cols is not None and dirty_from is None and self.n == n:
            return True
        tail = blocks[keep:]
        cols = hb = ho = None
        if keep and tail:
            tcols, thb, tho = self._marshal(tail)
            merged = [self._concat(a, b, keep) for a, b in zip(self.cols, tcols)]
            if all(m is not None for m in merged):
                cols = merged
                end = int(self.hash_off[keep])
                hb = np.concatenate([self.hash_blob[:end], thb]); ho = np.concatenate([self.hash_off[:keep + 1], tho[1:] + np.uint64(end)])
                self.marshalled = len(tail)
        if cols is None:
            cols, hb, ho = self._marshal(blocks)
            self.marshalled = n
        if cols[4].tag is not None or cols[4].uniform != _abi.J_STR:
            return False                                    # previous_hash values that are not strings: not resident
        arr = _cols_struct(cols)
        _abi.check(_abi.lib().fei_chain_load_cols(self.h, arr, _abi.ptr(np.ascontiguousarray(hb)), _abi.ptr(np.ascontiguousarray(ho)), n, 0))
        self.cols, self.hash_blob, self.hash_off, self.n = cols, hb, ho, n
        self.uploads += 1
        return True

    def validate(self) -> Tuple[int, int]:
        fb, kind = C.c_int64(-1), C.c_int32(0)
        _abi.check(_abi.lib().fei_chain_validate(self.h, C.byref(fb), C.byref(kind), None, None))
        return fb.value, kind.value


class MemoryChain:
    """The ledger slice of the reference's ``MemoryChain``: building (genesis, add_memory with GPU proof of work), validating
    (:596-618), syncing (receive_chain_update) and persisting (serialize / save / load) a chain.

    Consensus voting, wallet and networking are out of scope (SURVEY.md section 2).  Unlike the reference constructor this one
    does not touch the disk: pass ``chain_file`` to have add_memory persist after every block as the reference does.
    """

    def __init__(self, node_id: str = "validator", difficulty: int = 2, blocks: Optional[Iterable[Any]] = None,
                 chain_file: Optional[str] = None):
        self.lock = threading.RLock()
        self._res: Optional[_Resident] = None
        self._dirty_from: Optional[int] = 0
        self._all_tracked = False
        self.chain = list(blocks) if blocks is not None else []
        self.node_id = node_id
        self.difficulty = difficulty
        self.chain_file = chain_file      # None: nothing is written behind the caller's back; save_chain() then uses CHAIN_FILE
        if len(self._chain) > 1:
            self._sync_resident()         # the device image is built when blocks arrive, not when they are first validated

    # `chain` stays a list for every caller; assignments and in-place edits are noticed
    @property
    def chain(self) -> List[Any]:
        return self._chain

    @chain.setter
    def chain(self, blocks: Iterable[Any]) -> None:
        self._chain = _TrackedList(self, blocks)
        self._dirty_from = 0

    def _touch(self, pos: int) -> None:
        self._dirty_from = pos if self._dirty_from is None else min(self._dirty_from, pos)
        if pos == 0:
            self._all_tracked = False

    def _sync_resident(self) -> bool:
        """Marshal what changed (blocks from the lowest touched index on), hand the columns to the GPU, start watching the blocks."""
        with self.lock:
            if os.environ.get("FEI_CHAIN_RESIDENT", "1") == "0":
                return False
            if self._res is None:
                self._res = _Resident()
            start = self._dirty_from
            try:
                ok = self._res.sync(self._chain, start)
            except NotImplementedError:
                ok = False
            if not ok:
                return False
            if start is not None:
                for pos in range(min(start, len(self._chain)), len(self._chain)):
                    _track(self._chain[pos], self, pos)
                self._all_tracked = (self._all_tracked or start == 0) and all(type(b) is _TrackedBlock for b in self._chain[start:])
            # blocks of other classes cannot report their own mutations: such a chain is marshalled afresh on every call
            self._dirty_from = None if self._all_tracked else 0
            return True

    def validate_chain(self) -> bool:
        """Reference :596-618.  The blocks' hashed fields live on the device as typed columns -> canonical JSON -> SHA-ready blocks
        (built when the blocks arrived; only blocks touched since are marshalled again), so a call is one GPU pass over resident data."""
        with self.lock:
            if len(self._chain) < 2:
                return True
            if not self._sync_resident():
                return validate_chain_blocks(self._chain, lock=self.lock, log=logger)
            first_bad, kind = self._res.validate()
        if first_bad < 0:
            return True
        logger.error(f"Block {first_bad} has invalid hash" if kind == 1 else f"Block {first_bad} has broken link to previous block")
        return False

    # ---- building and persisting the ledger (reference :528-594, :1130-1172); proof of work runs on the GPU (mine_block)
    def create_genesis_block(self) -> None:
        """Reference :528-550 (same memory payload; the date object is kept in memory_data exactly as there)."""
        from datetime import datetime
        genesis_memory = {
            "metadata": {"unique_id": "genesis", "timestamp": time.time(), "date": datetime.now(), "flags": []},
            "headers": {"Subject": "Genesis Block", "Tags": "system,genesis,memorychain", "Status": "system"},
            "content": "Initial block of the Memory Chain. Created on " + datetime.now().isoformat(),
        }
        genesis_block = MemoryBlock(0, time.time(), genesis_memory, "0", self.node_id, self.node_id)
        genesis_block.mine_block(self.difficulty)
        with self.lock:
            self.chain.append(genesis_block)

    def get_latest_block(self) -> "MemoryBlock":
        with self.lock:
            return self.chain[-1]

    def add_memory(self, memory_data: Dict[str, Any], responsible_node: Optional[str] = None) -> str:
        """Reference :562-594: link to the latest block, mine (GPU nonce search), append, persist.  Returns the new hash."""
        if responsible_node is None:
            responsible_node = self.node_id
        previous_block = self.get_latest_block()
        new_block = MemoryBlock(previous_block.index + 1, time.time(), memory_data, previous_block.hash,
                                responsible_node, self.node_id)
        new_block.mine_block(self.difficulty)
        with self.lock:
            self.chain.append(new_block)
            if self.chain_file:
                self.save_chain()
            if len(self._chain) > 1:
                self._sync_resident()     # the new block joins the device image now (one block marshalled)
        return new_block.hash

    def serialize_chain(self) -> List[Dict[str, Any]]:
        with self.lock:
            return [block.to_dict() for block in self.chain]

    def save_chain(self) -> None:
        """Reference :1140-1149 (`json.dump(chain_data, f, indent=2)`), to `self.chain_file` (default: the reference's CHAIN_FILE)."""
        with self.lock:
            chain_data = self.serialize_chain()
            path = self.chain_file or CHAIN_FILE
            os.makedirs(os.path.dirname(path), exist_ok=True)
            with open(path, "w") as f:
                json.dump(chain_data, f, indent=2)

    def load_chain(self) -> bool:
        """Reference :1151-1172: True when a non-empty chain was read."""
        path = self.chain_file or CHAIN_FILE
        try:
            if not os.path.exists(path):
                return False
            with open(path, "r") as f:
                chain_data = json.load(f)
            with self.lock:
                self.chain = [MemoryBlock.from_dict(block_data) for block_data in chain_data]
                if len(self._chain) > 1:
                    self._sync_resident()
            return len(self.chain) > 0
        except (json.JSONDecodeError, KeyError, FileNotFoundError) as e:
            logger.error(f"Error loading chain: {e}")
            return False

    def receive_chain_update(self, chain_data: List[Dict[str, Any]]) -> bool:
        """Validation half of the reference's chain sync (:1037-1085): the same two checks as
        validate_chain (one GPU pass, log level warning), then the prefix test against the local chain.
        Persisting the accepted chain (save_chain) is the caller's business (out of scope here)."""
        new_chain = [MemoryBlock.from_dict(d) for d in chain_data]
        if len(new_chain) <= len(self.chain):
            logger.info("Received chain is not longer than current chain, ignoring")
            return False
        if len(new_chain) > 1:
            first_bad, kind, _ = hash_and_validate(new_chain)
            if first_bad >= 0:
                what = "has invalid hash" if kind == 1 else "has broken link to previous block"
                logger.warning(f"Rejecting chain update: Block {first_bad} {what}")
                return False
        with self.lock:
            for mine, theirs in zip(self.chain, new_chain):
                if mine.hash != theirs.hash:
                    logger.warning("Rejecting chain update: Chains have diverged")
                    return False
            self.chain = new_chain
            self._sync_resident()
        logger.info(f"Chain updated to {len(self.chain)} blocks")
        return True


def install(target_module: Any = None) -> None:
    """Patch the reference's class in place: ``memdir_tools.memorychain.MemoryChain.validate_chain``."""
    if target_module is None:
        import importlib
        target_module = importlib.import_module("memdir_tools.memorychain")

    def validate_chain(self) -> bool:
        return validate_chain_blocks(self.chain, lock=self.lock, log=target_module.logger)

    target_module.MemoryChain.validate_chain = validate_chain
