# coding: utf-8
"""Static checks on the compiled library (no GPU): the hot kernels exist for sm_90a with the
register / spill budget the design relies on, and their SASS holds the instructions the design
claims (check `cuobjdump` before spending GPU time):
  K1  FMNMX (ALU pipe) next to the IMAD pairs that carry half of the comparators on the FMA pipe;
  K2  TMA bulk copies (UBLKCP) + mbarrier waits (SYNCS) and the fp32 FADD / FFMA of the pairs;
  K6  one pass: no second kernel, a ticketed last-CTA reduction (ATOMG / RED on the counter).
Skipped when cuobjdump is not installed."""

import re
import shutil
import subprocess

import pytest

from byzantinemomentum_b200 import _lib

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
pytestmark = pytest.mark.skipif(shutil.which(CUOBJDUMP) is None, reason="cuobjdump not available")

def _run(*args):
  return subprocess.run([CUOBJDUMP, *args, str(_lib.library_path())], capture_output=True, text=True, timeout=600).stdout

@pytest.fixture(scope="module")
def usage():
  text = _run("-res-usage")
  table = {}
  for name, regs, stack in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)", text):
    table[name] = (int(regs), int(stack))
  assert len(table) > 400, "resource table not parsed"
  return table

def _find(usage, fragment):
  names = [k for k in usage if fragment in k]
  assert names, f"no kernel matching {fragment}"
  return names

def test_library_is_sm_90a_only():
  elf = _run("-lelf")
  archs = set(re.findall(r"sm_(\d+a?)", elf))
  assert archs == {"90a"}, archs

def test_register_and_spill_budgets(usage):
  # headline kernel: trimmed mean n = 25, f = 10, VEC = 4 -> 128 registers (4 CTAs of 128 threads per SM), no spill
  (headline,) = _find(usage, "k1_sortedILi25ELi4ELi10ELi0E")
  assert usage[headline] == (128, 0)
  # every specialised K1 kernel of the hot n stays spill free
  for n in (11, 25, 51):
    for name in _find(usage, f"k1_sortedILi{n}E"):
      if "ELin1E" in name:
        continue                                   # run-time f variants may keep a small frame
      assert usage[name][1] <= (32 if n == 51 else 0), (name, usage[name])   # n = 51: a few kernels keep a <= 32-byte frame
  for name in _find(usage, "k1_medianILi25E") + _find(usage, "k1_medianILi11E") + _find(usage, "k1_medianILi51E"):
    assert usage[name][0] <= 128 and usage[name][1] == 0, (name, usage[name])
  # one 512-thread CTA per SM for K2: at most 128 registers, no spill
  for name in _find(usage, "k2_pairdist"):
    assert usage[name][0] <= 128 and usage[name][1] == 0, (name, usage[name])
  for name in _find(usage, "k3_average") + _find(usage, "k4_bulyan_static"):
    assert usage[name][1] == 0, (name, usage[name])
  for name in _find(usage, "k6_study"):
    assert usage[name][1] <= 32, (name, usage[name])

def _sass(function):
  return _run("-sass", "-fun", function)

def test_k1_uses_both_pipes(usage):
  (headline,) = _find(usage, "k1_sortedILi25ELi4ELi10ELi0E")
  sass = _sass(headline)
  fmnmx = len(re.findall(r"\bFMNMX", sass))
  imad = len(re.findall(r"\bIMAD\b(?!\.MOV|\.WIDE|\.SHL|\.IADD|\.U32|\.HI)", sass))
  assert fmnmx > 300 and imad > 300, (fmnmx, imad)     # 4 columns per thread, comparators split over ALU and FMA pipes
  assert "LDG.E.128" in sass or "LDG.E.EF.128" in sass or re.search(r"LDG\.E\.[A-Z.]*128", sass)

def test_k2_stages_with_tma_and_computes_in_fp32(usage):
  names = _find(usage, "k2_pairdist_tmaILi4E")
  sass = _sass(names[0])
  assert "UBLKCP" in sass, "no TMA bulk copy in K2"
  assert "SYNCS" in sass, "no mbarrier in K2"
  # sm_90 has no packed fp32: each coordinate pair is two FADD and two FFMA (the unrolled 5 x 5 block)
  assert len(re.findall(r"\bFFMA\b", sass)) >= 200 and len(re.findall(r"\bFADD\b", sass)) >= 200
  assert "LDS.128" in sass

def test_k6_is_one_pass_with_a_ticketed_reduction(usage):
  names = _find(usage, "k6_studyILi32ELi2E")
  sass = _sass(names[0])
  assert re.search(r"\b(ATOMG|RED|ATOM)\.", sass), "no atomic (ticket / abs-max) in K6"
  assert "MEMBAR" in sass or "FENCE" in sass or "ERRBAR" in sass
