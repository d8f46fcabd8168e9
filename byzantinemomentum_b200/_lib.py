# coding: utf-8
"""ctypes binding of `libbyzagg.so` (C ABI: `include/byzagg.h`, `include/byzagg_shards.h` and
`include/byzagg_attack.h`).

The library is loaded lazily, on the first call that needs it, and the load FAILS LOUDLY:
there is no CPU or PyTorch fallback anywhere in this package.  Build it in-tree with
`python -c "import __graft_entry__ as g; g.build()"` or `make -C byzantinemomentum_b200/csrc`.
"""

import ctypes
import os
import pathlib
import threading

__all__ = ["lib", "LibraryError", "library_path", "check", "MAX_N", "STATUS_MESSAGES",
           "AKSEL_MODES", "STATUS_NO_FINITE_SET", "STATUS_DEGENERATE"]

MAX_N = 64
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

_lock = threading.Lock()
_lib = None

def lib():
  """ The loaded library (loads it on first use). """
  global _lib
  if _lib is not None:
    return _lib
  with _lock:
    if _lib is None:
      path = library_path()
      if not path.exists():
        raise LibraryError(f"{path} not found: build the CUDA extension first (python -c 'import __graft_entry__ as g; g.build()'); "
                           "this package has no CPU fallback")
      try:
        handle = ctypes.CDLL(str(path))
      except OSError as err:
        raise LibraryError(f"unable to load {path}: {err}") from err
      for name, (restype, argtypes) in list(SIGNATURES.items()) + list(SHARD_SIGNATURES.items()) + list(ATTACK_SIGNATURES.items()):
        try:
          fn = getattr(handle, name)
        except AttributeError as err:
          raise LibraryError(f"{path} does not export {name!r} (stale build?)") from err
        fn.restype = restype
        fn.argtypes = argtypes
      _lib = handle
  return _lib

def check(code, what):
  """ Raise on a non-zero return code of a bz_* call. """
  if code == 0:
    return
  message = lib().bz_last_error()
  message = message.decode("utf-8", "replace") if message else ""
  kinds = {-1: "invalid argument", -2: "unsupported", -3: "CUDA error", -4: "workspace"}
  error = ValueError if code in (-1, -2) else LibraryError
  raise error(f"{what} failed ({kinds.get(code, code)}): {message}")
