"""Patch an importable reference `memdir_tools` package in place so its callers (fei.tools.*, the Flask server,
the CLIs) run the hot path on the GPU without any source change:

    import fei_b200.dropin; fei_b200.dropin.install()

replaces  memdir_tools.search.search_memories          (search.py:337)
          memdir_tools.utils.search_memories           (utils.py:299, the legacy substring search)
          memdir_tools.filter.FilterManager.process_memories / run_filters   (filter.py:188, :311)
          memdir_tools.filter.MemoryFilter.matches     (filter.py:67)
          memdir_tools.memorychain.MemoryChain.validate_chain                (memorychain.py:596)
          memdir_tools.archiver.MemoryArchiver: archive_old_memories, cleanup_memories, empty_trash,
              apply_retention_policies, update_memory_statuses, run_maintenance   (archiver.py:205-639)
          memdir_tools.folders.MemdirFolderManager: get_folder_stats, list_folders, bulk_tag_folder   (folders.py:216-587)
          memdir_tools.cli: list_memories_cmd, view_memory, move_memory_cmd, search_memories_cmd, flag_memory   (cli.py:103-268)
          memdir_tools.search.main                      (search.py:596, what `python -m memdir_tools search` calls)
and adds  memdir_tools.filter.apply_filters.  Names other modules already imported (`from memdir_tools.search import
search_memories` in server.py / cli.py, the package's own re-exports) are rebound too, by identity.
Everything else of the reference (SearchQuery objects, MemoryFilter objects, MemoryArchiver settings, block classes,
servers) is used as is: the GPU layer only reads their public attributes."""
from __future__ import annotations

import importlib
import sys
from typing import Any


def _rebind(orig: Any, new: Any) -> None:
    """Point every module-level name that still holds `orig` (a `from x import f` done before install) at `new`."""
    for mod in list(sys.modules.values()):
        d = getattr(mod, "__dict__", None)
        if not d:
            continue
        for name, val in list(d.items()):
            if val is orig:
                d[name] = new


_ARCHIVER_STATE = ("archive_rules", "tag_based_archiving", "retention_policies", "cleanup_rules", "archive_folder", "trash_folder",
                   "archive_age", "trash_age")


def _install_archiver(cls: Any, sync_base) -> None:
    """The maintenance methods of the reference's MemoryArchiver run on the GPU against the reference object's settings.  The
    rule lists and dicts are shared, not copied, so the default rules a stage adds land on the reference object as there."""
    from .memdir_tools import archiver as garchiver

    def gpu(ref: Any) -> "garchiver.MemoryArchiver":
        sync_base()
        g = garchiver.MemoryArchiver()
        for name in _ARCHIVER_STATE:
            setattr(g, name, getattr(ref, name))
        return g

    def archive_old_memories(self, dry_run=False):
        return gpu(self).archive_old_memories(dry_run)

    def cleanup_memories(self, dry_run=False):
        return gpu(self).cleanup_memories(dry_run)

    def empty_trash(self, age_days=None, dry_run=False):
        return gpu(self).empty_trash(age_days, dry_run)

    def apply_retention_policies(self, dry_run=False):
        return gpu(self).apply_retention_policies(dry_run)

    def update_memory_statuses(self, dry_run=False):
        return gpu(self).update_memory_statuses(dry_run)

    def run_maintenance(self, dry_run=False):
        return {"archive": self.archive_old_memories(dry_run), "cleanup": self.cleanup_memories(dry_run),
                "trash": self.empty_trash(dry_run=dry_run), "retention": self.apply_retention_policies(dry_run),
                "status": self.update_memory_statuses(dry_run)}

    for fn in (archive_old_memories, cleanup_memories, empty_trash, apply_retention_policies, update_memory_statuses, run_maintenance):
        setattr(cls, fn.__name__, fn)


def _install_folders(cls: Any, sync_base) -> None:
    """The folder manager's whole-folder reads run on the GPU; the manager's file-system methods stay the reference's."""
    from .memdir_tools import folders as gfolders

    def gpu() -> "gfolders.MemdirFolderManager":
        sync_base()
        return object.__new__(gfolders.MemdirFolderManager)      # the reference object's __init__ already made the tree

    def get_folder_stats(self, folder_path, include_subfolders=False):
        return gpu().get_folder_stats(folder_path, include_subfolders)

    def list_folders(self, parent_folder="", recursive=False):
        return gpu().list_folders(parent_folder, recursive)

    def bulk_tag_folder(self, folder_path, tags, statuses=None, operation="add"):
        return gpu().bulk_tag_folder(folder_path, tags, statuses, operation)

    for fn in (get_folder_stats, list_folders, bulk_tag_folder):
        setattr(cls, fn.__name__, fn)


def _install_functions(ref_mod: Any, gpu_mod: Any, names, sync_base) -> None:
    """Module-level functions of the reference that run their GPU namesake against the reference's tree."""
    for name in names:
        fn = getattr(gpu_mod, name)

        def run(*a, _fn=fn, **k):
            sync_base()
            return _fn(*a, **k)
        run.__name__ = run.__qualname__ = name
        _rebind(getattr(ref_mod, name), run)
        setattr(ref_mod, name, run)


def install(package: str = "memdir_tools") -> None:
    ref_utils = importlib.import_module(f"{package}.utils")
    ref_search = importlib.import_module(f"{package}.search")
    ref_filter = importlib.import_module(f"{package}.filter")
    from .memdir_tools import filter as gfilter, search as gsearch, utils as gutils

    def _sync_base() -> None:
        gutils.set_memdir_base(ref_utils.MEMDIR_BASE)        # the tree the reference would walk (utils.py:16)

    def search_memories(query, folders=None, statuses=None, debug=False):
        _sync_base()
        return gsearch.search_memories(query, folders, statuses, debug)

    def _gpu_manager(mgr: Any) -> "gfilter.FilterManager":
        out = gfilter.FilterManager()
        for f in mgr.filters:
            g = gfilter.MemoryFilter(f.name)
            g.conditions, g.actions = f.conditions, f.actions
            out.add_filter(g)
        return out

    def process_memories(self, folders=None, statuses=None, dry_run=False):
        _sync_base()
        return _gpu_manager(self).process_memories(folders, statuses, dry_run)

    def matches(self, memory):
        g = gfilter.MemoryFilter(self.name)
        g.conditions = self.conditions
        return g.matches(memory)

    def run_filters(dry_run=False):
        _sync_base()
        return gfilter.run_filters(dry_run)

    def apply_filters(filters=None, folders=None, statuses=None, dry_run=False):
        _sync_base()
        if filters is not None and not isinstance(filters, gfilter.FilterManager) and hasattr(filters, "filters"):
            filters = _gpu_manager(filters)
        return gfilter.apply_filters(filters, folders, statuses, dry_run)

    def legacy_search_memories(query, folders=None, statuses=None, headers_only=False):
        _sync_base()
        return gutils.search_memories(query, folders, statuses, headers_only)

    _rebind(ref_search.search_memories, search_memories)
    ref_search.search_memories = search_memories
    _rebind(ref_utils.search_memories, legacy_search_memories)
    ref_utils.search_memories = legacy_search_memories
    ref_filter.FilterManager.process_memories = process_memories
    ref_filter.MemoryFilter.matches = matches
    _rebind(ref_filter.run_filters, run_filters)
    ref_filter.run_filters = run_filters
    ref_filter.apply_filters = apply_filters
    try:
        ref_arch = importlib.import_module(f"{package}.archiver")
    except ImportError:
        ref_arch = None
    if ref_arch is not None:
        _install_archiver(ref_arch.MemoryArchiver, _sync_base)
    try:
        ref_folders = importlib.import_module(f"{package}.folders")
    except ImportError:
        ref_folders = None
    if ref_folders is not None:
        _install_folders(ref_folders.MemdirFolderManager, _sync_base)
    try:
        ref_cli = importlib.import_module(f"{package}.cli")
    except ImportError:
        ref_cli = None
    if ref_cli is not None:                                 # the command line's listing, lookup and search commands; create / mkdir stay
        from .memdir_tools import cli as gcli
        _install_functions(ref_cli, gcli, ("list_memories_cmd", "view_memory", "move_memory_cmd", "search_memories_cmd", "flag_memory"),
                           _sync_base)
    if hasattr(ref_search, "main"):
        _install_functions(ref_search, gsearch, ("main",), _sync_base)
    try:
        ref_chain = importlib.import_module(f"{package}.memorychain")
    except Exception:                                        # the reference module needs `requests`
        ref_chain = None
    if ref_chain is not None:
        from .memdir_tools.memorychain import install as install_chain
        install_chain(ref_chain)
