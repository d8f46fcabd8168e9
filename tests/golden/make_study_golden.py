#!/usr/bin/env python3
# coding: utf-8
"""Generate `tests/golden/study_avg_dev_max.npz`: outputs of the UNMODIFIED reference's
`tools.compute_avg_dev_max` (tools/pytorch.py:97-125) on the input rows of every existing
`golden_*.npz` fixture, split the way attack.py:846-848 calls it: all rows ("sampled"),
the honest rows, the Byzantine rows (which may be an empty list).

Run with $BYZ_REFERENCE set to the root of a ByzantineMomentum checkout:

    python tests/golden/make_study_golden.py
"""

import json
import os
import pathlib
import sys

import numpy as np
import torch

REF = os.environ["BYZ_REFERENCE"]
sys.path.insert(0, REF)
_stdout, _stderr, _hook = sys.stdout, sys.stderr, sys.excepthook
import tools  # noqa: E402  (wraps stdout/stderr at import: tools/__init__.py:215-216,246)
sys.stdout, sys.stderr, sys.excepthook = _stdout, _stderr, _hook

HERE = pathlib.Path(__file__).resolve().parent

def main():
  torch.set_num_threads(1)
  data, cases = {}, []
  for path in sorted(HERE.glob("golden_*.npz")):
    z = np.load(path, allow_pickle=False)
    manifest = json.loads(str(z["manifest"]))
    rows = z["rows"]
    n, nb = manifest["n"], manifest["nb_byz"]
    splits = {"sampled": (0, n), "honest": (0, n - nb), "attack": (n - nb, n)}
    for split, (lo, hi) in splits.items():
      samples = [torch.from_numpy(rows[i].copy()) for i in range(lo, hi)]
      avg, norm_avg, norm_dev, norm_max = tools.compute_avg_dev_max(samples)
      tag = f"{manifest['name']}/{split}"
      if avg is not None:
        data[tag + "/avg"] = avg.numpy()
      cases.append(dict(fixture=path.name, split=split, lo=lo, hi=hi, tag=tag, has_avg=avg is not None,
                        norm_avg=repr(float(norm_avg)), norm_dev=repr(float(norm_dev)), norm_max=repr(float(norm_max))))
  data["manifest"] = np.array(json.dumps(dict(torch=torch.__version__, numpy=np.__version__, threads=1,
                                              function="tools.compute_avg_dev_max", cases=cases)))
  out = HERE / "study_avg_dev_max.npz"
  np.savez_compressed(out, **data)
  print(f"{out}: {len(cases)} cases, {out.stat().st_size} bytes")

if __name__ == "__main__":
  main()
