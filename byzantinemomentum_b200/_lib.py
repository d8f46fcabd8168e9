# coding: utf-8
"""ctypes binding of `libbyzagg.so` (C ABI: `include/byzagg.h`, `include/byzagg_shards.h`,
`include/byzagg_attack.h`, `include/byzagg_search_shards.h`, `include/byzagg_search_peers.h`,
`include/byzagg_coordinate.h`, `include/byzagg_peers_next.h`, `include/byzagg_distance.h`,
`include/byzagg_distance_shards.h`, `include/byzagg_anticge.h`, `include/byzagg_anticge_peers.h` and
`include/byzagg_distance_search.h` and `include/byzagg_distance_search_shards.h`), of the
second library `libbyzagg_peers.so` built next to it (C ABI: `include/byzagg_distance_peers.h`) and of the third,
`libbyzagg_star.so` (C ABI: `include/byzagg_rowshare_star.h`), which the callers compose with the first through their
C ABIs, of the fourth, `libbyzagg_many.so` (C ABI: `include/byzagg_coordinate_many.h`), which links against the first, and of
the fifth, `libbyzagg_many_tools.so` (C ABI: `include/byzagg_many_tools.h`), which links against the first and the fourth,
of the sixth, `libbyzagg_many_distance.so` (C ABI: `include/byzagg_distance_many.h` and
`include/byzagg_distance_many_table.h`), which links against the first and the fourth, and of the seventh,
`libbyzagg_many_search.so` (C ABI: `include/byzagg_distance_search_many.h`), which links against the first, the fourth and
the sixth.

Each library is loaded lazily, on the first call that needs it, and the load FAILS LOUDLY:
there is no CPU or PyTorch fallback anywhere in this package.  Build it in-tree with
`python -c "import __graft_entry__ as g; g.build()"` or `make -C byzantinemomentum_b200/csrc`.
"""

import ctypes
import os
import pathlib
import threading

__all__ = ["lib", "peers_lib", "star_lib", "many_lib", "many_tools_lib", "many_distance_lib", "many_search_lib", "LibraryError", "library_path",
           "peers_library_path", "star_library_path", "many_library_path", "many_tools_library_path", "many_distance_library_path", "many_search_library_path", "check", "MAX_N", "MAX_N_COORDINATE", "MAX_N_MANY", "MAX_N_DISTANCE", "STATUS_MESSAGES",
           "AKSEL_MODES", "STATUS_NO_FINITE_SET", "STATUS_DEGENERATE"]

MAX_N = 64
MAX_N_COORDINATE = 128      # BZ_MAX_N_COORDINATE: the coordinate-wise rules through bz_coordinate
MAX_N_MANY = 1024           # BZ_MAX_N_MANY: the coordinate-wise rules through bz_coordinate_many
MAX_N_DISTANCE = 128        # BZ_MAX_N_DISTANCE: Multi-Krum, Bulyan, Aksel and CGE through bz_distance
MAX_PEERS = 16
STATUS_NO_FINITE_SET = 1
STATUS_DEGENERATE = 2
STATUS_PEER_TIMEOUT = 3
STATUS_MESSAGES = {
  STATUS_NO_FINITE_SET: "Too many non-finite gradients: a non-Byzantine gradient must only contain finite coordinates",
  STATUS_DEGENERATE: "Too many non-finite scores: fewer finite Multi-Krum scores than gradients to average",
}
AKSEL_MODES = {"mid": 0, "n-f": 1}

class LibraryError(RuntimeError):
  """ The CUDA library is missing, fails to load, or reported an error. """

def library_path():
  override = os.environ.get("BYZAGG_LIBRARY")
  if override:
    return pathlib.Path(override)
  return pathlib.Path(__file__).resolve().parent / "libbyzagg.so"

def peers_library_path():
  """ libbyzagg_peers.so: next to libbyzagg.so, or where BYZAGG_PEERS_LIBRARY says. """
  override = os.environ.get("BYZAGG_PEERS_LIBRARY")
  if override:
    return pathlib.Path(override)
  return library_path().parent / "libbyzagg_peers.so"

def star_library_path():
  """ libbyzagg_star.so: next to libbyzagg.so, or where BYZAGG_STAR_LIBRARY says. """
  override = os.environ.get("BYZAGG_STAR_LIBRARY")
  if override:
    return pathlib.Path(override)
  return library_path().parent / "libbyzagg_star.so"

def many_library_path():
  """ libbyzagg_many.so: next to libbyzagg.so, or where BYZAGG_MANY_LIBRARY says. """
  override = os.environ.get("BYZAGG_MANY_LIBRARY")
  if override:
    return pathlib.Path(override)
  return library_path().parent / "libbyzagg_many.so"

def many_tools_library_path():
  """ libbyzagg_many_tools.so: next to libbyzagg.so, or where BYZAGG_MANY_TOOLS_LIBRARY says. """
  override = os.environ.get("BYZAGG_MANY_TOOLS_LIBRARY")
  if override:
    return pathlib.Path(override)
  return library_path().parent / "libbyzagg_many_tools.so"

def many_distance_library_path():
  """ libbyzagg_many_distance.so: next to libbyzagg.so, or where BYZAGG_MANY_DISTANCE_LIBRARY says. """
  override = os.environ.get("BYZAGG_MANY_DISTANCE_LIBRARY")
  if override:
    return pathlib.Path(override)
  return library_path().parent / "libbyzagg_many_distance.so"

def many_search_library_path():
  """ libbyzagg_many_search.so: next to libbyzagg.so, or where BYZAGG_MANY_SEARCH_LIBRARY says. """
  override = os.environ.get("BYZAGG_MANY_SEARCH_LIBRARY")
  if override:
    return pathlib.Path(override)
  return library_path().parent / "libbyzagg_many_search.so"

_c_rows = ctypes.POINTER(ctypes.c_void_p)
_vp, _i, _i64, _sz, _dbl = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_size_t, ctypes.c_double

# name -> (restype, argtypes); must list every symbol of include/byzagg.h (tests check it)
SIGNATURES = {
  "bz_version": (_i, []),
  "bz_max_n": (_i, []),
  "bz_last_error": (ctypes.c_char_p, []),
  "bz_workspace_bytes": (_sz, [_i]),
  "bz_average": (_i, [_c_rows, _i, _i64, _vp, _vp]),
  "bz_median": (_i, [_c_rows, _i, _i64, _vp, _vp]),
  "bz_trmean": (_i, [_c_rows, _i, _i, _i64, _vp, _vp]),
  "bz_phocas": (_i, [_c_rows, _i, _i, _i64, _vp, _vp]),
  "bz_meamed": (_i, [_c_rows, _i, _i, _i64, _vp, _vp]),
  "bz_krum": (_i, [_c_rows, _i, _i, _i, _i64, _vp, _vp, _vp, _sz, _vp]),
  "bz_bulyan": (_i, [_c_rows, _i, _i, _i, _i64, _vp, _vp, _vp, _vp, _sz, _vp]),
  "bz_brute": (_i, [_c_rows, _i, _i, _i64, _vp, _vp, _vp, _vp, _sz, _vp]),
  "bz_krum_reuse": (_i, [_c_rows, _i, _i, _i, _i64, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _sz, _vp]),
  "bz_bulyan_reuse": (_i, [_c_rows, _i, _i, _i, _i64, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _sz, _vp]),
  "bz_brute_reuse": (_i, [_c_rows, _i, _i, _i64, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _sz, _vp]),
  "bz_krum_peers": (_i, [_c_rows, _i, _i, _i, _i64, _vp, _vp, _vp, _i, _i, _c_rows, _c_rows, ctypes.c_uint, _vp, _sz, _vp]),
  "bz_bulyan_peers": (_i, [_c_rows, _i, _i, _i, _i64, _vp, _vp, _vp, _i, _i, _c_rows, _c_rows, ctypes.c_uint, _vp, _sz, _vp]),
  "bz_aksel": (_i, [_c_rows, _i, _i, _i, _i64, _vp, _vp, _vp, _sz, _vp]),
  "bz_cge": (_i, [_c_rows, _i, _i, _i64, _vp, _vp, _vp, _sz, _vp]),
  "bz_pairdist_partial": (_i, [_c_rows, _i, _i64, _vp, _vp, _sz, _vp]),
  "bz_rowdist_partial": (_i, [_c_rows, _i, _vp, _i64, _vp, _vp, _sz, _vp]),
  "bz_krum_select": (_i, [_vp, _i, _i, _i, _vp, _vp]),
  "bz_bulyan_select": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp]),
  "bz_brute_select": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp]),
  "bz_rowdist_select": (_i, [_vp, _i, _i, _i, _vp, _vp]),
  "bz_krum_select_peers": (_i, [_c_rows, _i, _i, _i, _vp, _vp]),
  "bz_bulyan_select_peers": (_i, [_c_rows, _i, _i, _i, _i, _vp, _vp, _vp]),
  "bz_brute_select_peers": (_i, [_c_rows, _i, _i, _i, _vp, _vp, _vp]),
  "bz_rowdist_select_peers": (_i, [_c_rows, _i, _i, _i, _vp, _vp]),
  "bz_avg_dev_max": (_i, [_c_rows, _i, _i64, _vp, _vp, _vp, _sz, _vp]),
  "bz_rowdots": (_i, [_c_rows, _i, _vp, _i64, _vp, _vp, _sz, _vp]),
  "bz_stage_rows": (_i, [_c_rows, _i, _i64, _vp, _i64, _vp]),
  "bz_coordinate_host": (_i, [_i, _c_rows, _i, _i, _i64, _vp, _vp, _i64, _vp, _i, _vp, _vp, _vp]),
  "bz_gradient_row": (_i, [_vp, _i64, _dbl, _vp, _i, _vp, _dbl, _dbl, _vp, _vp, _sz, _vp]),
  "bz_average_selected": (_i, [_c_rows, _i, _vp, _i, _i, _dbl, _vp, _i64, _vp, _vp]),
  "bz_bulyan_reduce": (_i, [_c_rows, _i, _i, _i, _vp, _vp, _i64, _vp, _vp]),
}

# the same for include/byzagg_shards.h (entry points of a d-sharded trainer besides the rules)
SHARD_SIGNATURES = {
  "bz_gradient_scatter": (_i, [_vp, _i64, _dbl, _i, _c_rows, _vp, _sz, _vp]),
  "bz_gradient_momentum": (_i, [_c_rows, _i, _i64, _i, _c_rows, _vp, _dbl, _dbl, _c_rows, _vp]),
}

# the same for include/byzagg_attack.h (the attacks' line search)
ATTACK_SIGNATURES = {
  "bz_line_search_workspace_bytes": (_sz, [_i]),
  "bz_line_search": (_i, [_i, _c_rows, _i, _i, _i, _i, _i, _vp, _vp, _i64, _i, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
}

# the same for include/byzagg_search_shards.h (the line search on a d-sharded trainer)
SEARCH_SHARD_SIGNATURES = {
  "bz_pairdist_partial_reuse": (_i, [_c_rows, _i, _i64, _vp, _vp, _vp, _i, _vp, _vp, _vp, _sz, _vp]),
  "bz_search_candidate": (_i, [_vp, _vp, _vp, _i64, _vp, _i, _i, _i, _vp]),
  "bz_search_score_partial": (_i, [_vp, _vp, _i64, _vp, _vp, _vp, _sz, _vp]),
  "bz_search_step": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _i, _i, _vp]),
}
# the same for include/byzagg_search_peers.h (that search with its exchanges over peer memory)
SEARCH_PEER_SIGNATURES = {
  "bz_pairdist_reuse_peers": (_i, [_i, _c_rows, _i, _i, _i, _i64, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _i, _i, _c_rows, _c_rows,
                                   ctypes.c_uint, _vp, _sz, _vp]),
  "bz_rowdist_peers": (_i, [_i, _c_rows, _i, _i, _i, _vp, _i64, _vp, _vp, _vp, _i, _i, _c_rows, _c_rows, ctypes.c_uint, _vp, _sz, _vp]),
  "bz_search_score_peers": (_i, [_vp, _vp, _i64, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _c_rows, _c_rows, ctypes.c_uint, _vp, _sz, _vp]),
}
# the same for include/byzagg_peers_next.h (the exchanges over peer memory with the epoch taken from the buffer)
PEER_NEXT_SIGNATURES = {
  "bz_krum_peers_next": (_i, [_c_rows, _i, _i, _i, _i64, _vp, _vp, _vp, _i, _i, _c_rows, _c_rows, _vp, _sz, _vp]),
  "bz_bulyan_peers_next": (_i, [_c_rows, _i, _i, _i, _i64, _vp, _vp, _vp, _i, _i, _c_rows, _c_rows, _vp, _sz, _vp]),
  "bz_pairdist_reuse_peers_next": (_i, [_i, _c_rows, _i, _i, _i, _i64, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _i, _i, _c_rows,
                                        _c_rows, _vp, _sz, _vp]),
  "bz_rowdist_peers_next": (_i, [_i, _c_rows, _i, _i, _i, _vp, _i64, _vp, _vp, _vp, _i, _i, _c_rows, _c_rows, _vp, _sz, _vp]),
  "bz_search_score_peers_next": (_i, [_vp, _vp, _i64, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _c_rows, _c_rows, _vp, _sz, _vp]),
}
# the same for include/byzagg_coordinate.h (the coordinate-wise rules up to MAX_N_COORDINATE rows)
COORDINATE_SIGNATURES = {
  "bz_coordinate": (_i, [_i, _c_rows, _i, _i, _i64, _vp, _vp]),
}
# the same for include/byzagg_coordinate_many.h, the table of the fourth library (`many_lib()`): the coordinate-wise
# rules up to MAX_N_MANY rows
COORDINATE_MANY_SIGNATURES = {
  "bz_coordinate_many_last_error": (ctypes.c_char_p, []),
  "bz_coordinate_many": (_i, [_i, _c_rows, _i, _i, _i64, _vp, _vp]),
}
# the same for include/byzagg_many_tools.h, the table of the fifth library (`many_tools_lib()`): the study metrics and the
# line search against the coordinate-wise rules up to MAX_N_MANY rows
MANY_TOOLS_SIGNATURES = {
  "bz_many_tools_last_error": (ctypes.c_char_p, []),
  "bz_avg_dev_max_many_workspace_bytes": (_sz, [_i]),
  "bz_avg_dev_max_many": (_i, [_c_rows, _i, _i64, _vp, _vp, _vp, _sz, _vp]),
  "bz_line_search_many_workspace_bytes": (_sz, [_i]),
  "bz_line_search_many": (_i, [_i, _c_rows, _i, _i, _i, _i, _i, _vp, _vp, _i64, _i, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
}
# the same for include/byzagg_distance_many.h, the table of the sixth library (`many_distance_lib()`): Multi-Krum, Bulyan,
# Aksel and CGE up to MAX_N_MANY rows
MANY_DISTANCE_SIGNATURES = {
  "bz_distance_many_last_error": (ctypes.c_char_p, []),
  "bz_distance_many_workspace_bytes": (_sz, [_i]),
  "bz_distance_many": (_i, [_i, _c_rows, _i, _i, _i, _i, _i64, _vp, _vp, _vp, _vp, _sz, _vp]),
}
# the same for include/byzagg_distance_many_table.h, also in the sixth library: the selection and reduce of Multi-Krum and
# Bulyan from the distance table `bz_distance_many` leaves in its workspace
MANY_DISTANCE_TABLE_SIGNATURES = {
  "bz_distance_many_select": (_i, [_i, _c_rows, _i, _i, _i, _i64, _vp, _vp, _vp, _vp, _sz, _vp]),
}
# the same for include/byzagg_distance_search_many.h, the table of the seventh library (`many_search_lib()`): the line
# search against Multi-Krum, Bulyan, Aksel and CGE up to MAX_N_MANY rows
MANY_SEARCH_SIGNATURES = {
  "bz_distance_line_search_many_last_error": (ctypes.c_char_p, []),
  "bz_distance_line_search_many_workspace_bytes": (_sz, [_i]),
  "bz_distance_line_search_many": (_i, [_i, _c_rows, _i, _i, _i, _i, _i, _vp, _vp, _i64, _i, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
}
# the same for include/byzagg_distance.h (Multi-Krum, Bulyan, Aksel and CGE up to MAX_N_DISTANCE rows)
DISTANCE_SIGNATURES = {
  "bz_distance_workspace_bytes": (_sz, [_i]),
  "bz_distance": (_i, [_i, _c_rows, _i, _i, _i, _i, _i64, _vp, _vp, _vp, _vp, _sz, _vp]),
}
# the same for include/byzagg_distance_shards.h (the d-sharded phases of those rules up to MAX_N_DISTANCE rows)
DISTANCE_SHARD_SIGNATURES = {
  "bz_distance_partial": (_i, [_i, _c_rows, _i, _vp, _i64, _vp, _vp, _sz, _vp]),
  "bz_distance_select": (_i, [_i, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
  "bz_distance_reduce": (_i, [_i, _c_rows, _i, _i, _i, _i, _vp, _vp, _i64, _vp, _vp]),
}
# the same for include/byzagg_anticge.h (the attack against CGE, on one GPU and on the d-sharded path)
ANTICGE_SIGNATURES = {
  "bz_anticge_workspace_bytes": (_sz, [_i]),
  "bz_anticge": (_i, [_c_rows, _i, _i, _i, _i64, _vp, _vp, _sz, _vp]),
  "bz_anticge_partial": (_i, [_c_rows, _i, _i, _vp, _i64, _vp, _vp, _vp, _sz, _vp]),
  "bz_anticge_scale": (_i, [_vp, _vp, _vp, _i, _i, _i, _i64, _vp, _vp]),
}
# the same for include/byzagg_anticge_peers.h (that attack on the d-sharded path with its exchanges over peer memory)
ANTICGE_PEER_SIGNATURES = {
  "bz_anticge_peers": (_i, [_c_rows, _i, _i, _i, _i64, _vp, _vp, _i, _i, _c_rows, _c_rows, ctypes.c_uint, _vp, _sz, _vp]),
  "bz_anticge_peers_next": (_i, [_c_rows, _i, _i, _i, _i64, _vp, _vp, _i, _i, _c_rows, _c_rows, _vp, _sz, _vp]),
}
# the same for include/byzagg_distance_search.h (the line search against Multi-Krum, Bulyan, Aksel and CGE up to
# MAX_N_DISTANCE rows)
DISTANCE_SEARCH_SIGNATURES = {
  "bz_distance_line_search_workspace_bytes": (_sz, [_i]),
  "bz_distance_line_search": (_i, [_i, _c_rows, _i, _i, _i, _i, _i, _vp, _vp, _i64, _i, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
}
# the same for include/byzagg_distance_search_shards.h (phase A of the d-sharded line search against Multi-Krum and
# Bulyan above MAX_N rows, with the honest rows' distances kept between evaluations)
DISTANCE_SEARCH_SHARD_SIGNATURES = {
  "bz_distance_pass_tables_bytes": (_sz, []),
  "bz_distance_partial_reuse": (_i, [_i, _c_rows, _i, _i64, _vp, _vp, _vp, _i, _vp, _vp, _vp, _sz, _vp]),
}
# the same for include/byzagg_distance_peers.h, the table of the second library (`peers_lib()`): phase B of the d-sharded
# distance rules above MAX_N rows with its exchange over peer memory
DISTANCE_PEER_SIGNATURES = {
  "bz_distance_peers_last_error": (ctypes.c_char_p, []),
  "bz_distance_select_peers": (_i, [_i, _vp, _i, _i, _i, _i, _vp, _vp, _i, _i, _c_rows, _c_rows, ctypes.c_uint, _vp]),
  "bz_distance_select_peers_next": (_i, [_i, _vp, _i, _i, _i, _i, _vp, _vp, _i, _i, _c_rows, _c_rows, _vp]),
}
# the same for include/byzagg_rowshare_star.h, the table of the third library (`star_lib()`): CGE's candidate-only
# phase A of the d-sharded line search above MAX_N rows
ROWSHARE_STAR_SIGNATURES = {
  "bz_rowshare_star_last_error": (ctypes.c_char_p, []),
  "bz_rowshare_star_workspace_bytes": (_sz, [_i]),
  "bz_rowshare_star": (_i, [_c_rows, _i, _i, _i64, _vp, _vp, _sz, _vp]),
}
SEARCH_STATE_BYTES = 64                     # BZ_SEARCH_STATE_BYTES
CANDIDATE_FIRST, CANDIDATE_NEXT, CANDIDATE_FINAL = 0, 1, 2

_lock = threading.Lock()
_lib = None
_peers_lib = None
_star_lib = None
_many_lib = None
_many_tools_lib = None
_many_distance_lib = None
_many_search_lib = None

def _load(path, tables):
  """ The library at `path` with the signatures of `tables` bound; LibraryError when it is missing or stale. """
  if not path.exists():
    raise LibraryError(f"{path} not found: build the CUDA extension first (python -c 'import __graft_entry__ as g; g.build()'); "
                       "this package has no CPU fallback")
  try:
    handle = ctypes.CDLL(str(path))
  except OSError as err:
    raise LibraryError(f"unable to load {path}: {err}") from err
  for name, (restype, argtypes) in [item for table in tables for item in table.items()]:
    try:
      fn = getattr(handle, name)
    except AttributeError as err:
      raise LibraryError(f"{path} does not export {name!r} (stale build?)") from err
    fn.restype = restype
    fn.argtypes = argtypes
  return handle

def lib():
  """ The loaded library (loads it on first use). """
  global _lib
  if _lib is not None:
    return _lib
  with _lock:
    if _lib is None:
      _lib = _load(library_path(), (SIGNATURES, SHARD_SIGNATURES, ATTACK_SIGNATURES, SEARCH_SHARD_SIGNATURES, SEARCH_PEER_SIGNATURES,
                                    COORDINATE_SIGNATURES, PEER_NEXT_SIGNATURES, DISTANCE_SIGNATURES, DISTANCE_SHARD_SIGNATURES,
                                    ANTICGE_SIGNATURES, ANTICGE_PEER_SIGNATURES, DISTANCE_SEARCH_SIGNATURES,
                                    DISTANCE_SEARCH_SHARD_SIGNATURES))
  return _lib

def peers_lib():
  """ The second library, libbyzagg_peers.so (loads it on first use; no fallback when it is missing). """
  global _peers_lib
  if _peers_lib is not None:
    return _peers_lib
  with _lock:
    if _peers_lib is None:
      _peers_lib = _load(peers_library_path(), (DISTANCE_PEER_SIGNATURES,))
  return _peers_lib

def star_lib():
  """ The third library, libbyzagg_star.so (loads it on first use; no fallback when it is missing). """
  global _star_lib
  if _star_lib is not None:
    return _star_lib
  with _lock:
    if _star_lib is None:
      _star_lib = _load(star_library_path(), (ROWSHARE_STAR_SIGNATURES,))
  return _star_lib

def many_lib():
  """ The fourth library, libbyzagg_many.so (loads it on first use; no fallback when it is missing). """
  global _many_lib
  if _many_lib is not None:
    return _many_lib
  lib()                          # libbyzagg.so first: the fourth library links against it
  with _lock:
    if _many_lib is None:
      _many_lib = _load(many_library_path(), (COORDINATE_MANY_SIGNATURES,))
  return _many_lib

def many_tools_lib():
  """ The fifth library, libbyzagg_many_tools.so (loads it on first use; no fallback when it is missing). """
  global _many_tools_lib
  if _many_tools_lib is not None:
    return _many_tools_lib
  many_lib()                     # libbyzagg.so and libbyzagg_many.so first: the fifth library links against both
  with _lock:
    if _many_tools_lib is None:
      _many_tools_lib = _load(many_tools_library_path(), (MANY_TOOLS_SIGNATURES,))
  return _many_tools_lib

def many_distance_lib():
  """ The sixth library, libbyzagg_many_distance.so (loads it on first use; no fallback when it is missing). """
  global _many_distance_lib
  if _many_distance_lib is not None:
    return _many_distance_lib
  many_lib()                     # libbyzagg.so and libbyzagg_many.so first: the sixth library links against both
  with _lock:
    if _many_distance_lib is None:
      _many_distance_lib = _load(many_distance_library_path(), (MANY_DISTANCE_SIGNATURES, MANY_DISTANCE_TABLE_SIGNATURES))
  return _many_distance_lib

def many_search_lib():
  """ The seventh library, libbyzagg_many_search.so (loads it on first use; no fallback when it is missing). """
  global _many_search_lib
  if _many_search_lib is not None:
    return _many_search_lib
  many_distance_lib()            # the first, fourth and sixth libraries first: the seventh links against them
  with _lock:
    if _many_search_lib is None:
      _many_search_lib = _load(many_search_library_path(), (MANY_SEARCH_SIGNATURES,))
  return _many_search_lib

def check(code, what):
  """ Raise on a non-zero return code of a bz_* call. """
  if code == 0:
    return
  # each library keeps the message of its own last failure
  if what in DISTANCE_PEER_SIGNATURES:
    message = peers_lib().bz_distance_peers_last_error()
  elif what in ROWSHARE_STAR_SIGNATURES:
    message = star_lib().bz_rowshare_star_last_error()
  elif what in COORDINATE_MANY_SIGNATURES:
    message = many_lib().bz_coordinate_many_last_error()
  elif what in MANY_TOOLS_SIGNATURES:
    message = many_tools_lib().bz_many_tools_last_error()
  elif what in MANY_DISTANCE_SIGNATURES or what in MANY_DISTANCE_TABLE_SIGNATURES:
    message = many_distance_lib().bz_distance_many_last_error()
  elif what in MANY_SEARCH_SIGNATURES:
    message = many_search_lib().bz_distance_line_search_many_last_error()
  else:
    message = lib().bz_last_error()
  message = message.decode("utf-8", "replace") if message else ""
  kinds = {-1: "invalid argument", -2: "unsupported", -3: "CUDA error", -4: "workspace"}
  error = ValueError if code in (-1, -2) else LibraryError
  raise error(f"{what} failed ({kinds.get(code, code)}): {message}")
