#!/usr/bin/env python3
# coding: utf-8
"""Opcode histogram of the hot kernels in libbyzagg.so (cuobjdump -sass), the tracked evidence that
the kernels are sm_90a code using TMA bulk copies (UBLKCP), mbarriers (SYNCS), fp32 FADD / FFMA,
dual-pipe comparators (FMNMX + IMAD) and no tensor-core instruction.
    python tools/sass_hist.py"""
import collections, pathlib, re, subprocess, sys
ROOT = pathlib.Path(__file__).resolve().parent.parent
lib = ROOT / "byzantinemomentum_b200" / "libbyzagg.so"
WANT = [r"k2_ringILi512ELi4ELb0ELb0", r"k2_ringILi512ELi4ELb1ELb0", r"k2_ringILi256ELi3ELb0ELb1", r"k1_sortedILi25ELi4ELi10ELi0", r"k1_medianILi25ELi4",
        r"k1_medianILi51ELi2", r"k3_averageILi4", r"k4_bulyan_staticILi25ELi5ELi2", r"k2_rowdistILb0ELi4", r"k6_studyILi32ELi2", r"k7_produceILi1"]
out = subprocess.run(["cuobjdump", "-sass", str(lib)], capture_output=True, text=True).stdout
arch = sorted(set(re.findall(r"arch = (sm_\w+)", out)))
print(f"# {lib.name}: architectures in the fat binary: {', '.join(arch)}")
funcs = re.split(r"\n\s*Function : ", out)
for pat in WANT:
  for f in funcs[1:]:
    name = f.split("\n", 1)[0].strip()
    if re.search(pat, name):
      ops = collections.Counter()
      for m in re.finditer(r"^\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d\s+)?([A-Z][A-Z0-9_]*)", f, re.M):
        ops[m.group(1)] += 1
      total = sum(ops.values())
      demangled = subprocess.run(["c++filt", name], capture_output=True, text=True).stdout.strip()
      print(f"\n## {demangled[:150]}\n   {total} SASS instructions; top opcodes: " + ", ".join(f"{o} {c}" for o, c in ops.most_common(14)))
      flags = {k: ops.get(k, 0) for k in ("UBLKCP", "SYNCS", "FADD", "FFMA", "FMNMX", "IMAD", "LDS", "LDG", "LDGSTS", "ATOM", "ATOMG", "RED", "HMMA", "HGMMA")}
      print("   markers: " + ", ".join(f"{k} {v}" for k, v in flags.items() if v or k in ("HMMA", "HGMMA")))
      break
