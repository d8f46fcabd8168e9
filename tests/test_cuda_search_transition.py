# coding: utf-8
"""GPU tests of the attacks' line search on scores its random-data tests never produce.

  * The transition itself (`bz_search_step`, K9, whose `search_step` the score passes of every search path
    share) driven directly through ctypes on the scripted scapes of tests/line_scapes.py, for evals 1 to
    40, 64 and 200, over 1, 2, 3, 8, 16 or 1000 score shares: shares whose sum depends on their rank
    order, sums half an fp32 ulp from two floats (round to even) and sums at fp32's overflow edge.  Every
    x_k, every y_k = fl32(((p0 + p1) + p2) + ...) and the chosen factor are those of
    tests/line_oracle.py fed the same y values, compared by `float.hex()`; the status word keeps the
    first non-zero evaluation status, is reset at k = 0 and takes a NULL status pointer.
  * K8 (`bz_search_candidate`) after each transition and at the end: the candidate row of the factor the
    state holds is the torch statement of the reference (`avg + s * att`, s = -x with `negative`;
    `avg.mul(-x)` for empire-strict; no sign on the final factor), bit for bit, on rows holding +-0,
    subnormals, +-inf, NaN and +-FLT_MAX, off the 16-byte grid, for d = 1, 3, 1031 and 70001.
  * Every search path on score landscapes built of exact ties, y = 0, NaN at x = 0 only, +inf from
    overflow and finite levels far apart (`_landscapes`), both candidate kinds, `negative` on and off:
    `engine.LineSearch` up to 64 rows for all ten rules and at 100 rows (`bz_line_search` for the
    coordinate-wise rules, `bz_distance_line_search` for Multi-Krum, Bulyan, Aksel and CGE),
    `ShardedLineSearch` with the collective exchange on 1 and 3 emulated ranks (and `wide=True` at 100
    rows), with the fused exchange on 2 emulated ranks and on one, and one graph replay per path.  The x
    sequence, the factor and `byz` are those of the reference's host loop over the plain rules, bit for
    bit with no tie tolerance, as are the scores that are 0 or not finite."""

import math

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
DEV = "cuda:0"

import line_oracle
import line_scapes
from line_scapes import FLT_MAX, FLT_MIN, FLT_TRUE_MIN, INF, NAN

NPARTS = [1, 2, 3, 8, 16, 1000]
GARBAGE_STATUS = 0x5A5A

def _lib():
  from byzantinemomentum_b200 import _lib
  return _lib

def _stream():
  return torch.cuda.current_stream().cuda_stream

def _fl32(y):
  with np.errstate(over="ignore"):
    return float(np.float32(y))

def _ulp32(w):
  """ The fp32 ulp of the finite fp32 value w (> 0). """
  w = abs(w)
  if w < FLT_MIN:
    return FLT_TRUE_MIN
  return 2. ** (math.frexp(w)[1] - 24)

# ---------------------------------------------------------------------------- #
# Score shares: P doubles for the scripted value v, the first P - 2 (or P - 1) of them -0.0, which leaves
# any sum as it is

def _plain(v, P):
  return [-0.] * (P - 1) + [v]

def _rank_order(v, P):
  """ 1e300 first, -1e300 and v last: added in rank order the sum is v; in any other order 1e300 and
  -1e300 absorb v first. """
  if P < 3:
    return _plain(v, P)
  return [1e300] + [-0.] * (P - 3) + [-1e300, v]

def _halfway(v, P):
  """ fl32(v) and half its fp32 ulp: a sum exactly between two fp32 values, which rounds to even. """
  w = _fl32(v)
  if P < 2 or not math.isfinite(w) or w == 0.:
    return _plain(v, P)
  return [-0.] * (P - 2) + [w, math.copysign(_ulp32(w) / 2, w)]

def _overflow_edge(v, P):
  """ FLT_MAX plus a share that puts the sum just below (v < 0: fl32 gives FLT_MAX), exactly at (v > 0)
  or just above (v = 0) FLT_MAX + ulp / 2, where fl32 rounds to inf; NaN stays NaN. """
  if P < 2:
    return _plain(v, P)
  half = 2. ** 103
  e = NAN if math.isnan(v) else half + 2. ** 76 if v == 0 else half if v > 0 else half - 2. ** 76
  return [-0.] * (P - 2) + [FLT_MAX, e]

SHARES = {"plain": _plain, "rank-order": _rank_order, "halfway": _halfway, "overflow-edge": _overflow_edge}

def _sum_in_rank_order(parts):
  total = parts[0]
  for p in parts[1:]:
    total += p
  return total

def _oracle(ys, extra=0.):
  """ (x sequence, factor) of line_maximize fed the scores ys, and the x a further evaluation would take. """
  xs = []
  factor = line_oracle.line_maximize(lambda x: (xs.append(x), ys[len(xs) - 1])[1], len(ys))
  more = []
  line_oracle.line_maximize(lambda x: (more.append(x), (ys + [extra])[len(more) - 1])[1], len(ys) + 1)
  return xs, factor, more[-1]

def _script(scape, evals, P, pattern):
  """ The shares of every evaluation (the scape reads the x the oracle evaluates) and the y values. """
  parts, ys = [], []
  def fed(x):
    k = len(ys)
    shares = SHARES[pattern](scape(k, x, evals), P)
    parts.append(shares)
    ys.append(_fl32(_sum_in_rank_order(shares)))
    return ys[-1]
  line_oracle.line_maximize(fed, evals)
  return parts, ys

def _status_words(evals, which):
  """ Per-evaluation status words: none (a NULL pointer), one non-zero word, or several (the first wins). """
  if which == "none":
    return None, 0
  words = [0] * evals
  if which == "one":
    words[evals // 3] = 2
    return words, 2
  for k, w in ((evals - 1, 5), (evals // 2, 3), (evals // 4, 1)):
    words[k] = w
  return words, words[min(k for k in range(evals) if words[k])]

class _Search:
  """ Device buffers of one scripted search, reused from one search to the next. """
  def __init__(self):
    self.state = torch.empty(_lib().SEARCH_STATE_BYTES // 8, dtype=torch.float64, device=DEV)
    self.parts = torch.empty(200 * 1000, dtype=torch.float64, device=DEV)
    self.words = torch.empty(200, dtype=torch.int32, device=DEV)
    self.trace = torch.empty(2 * 200 + 1, dtype=torch.float64, device=DEV)
    self.status = torch.empty(1, dtype=torch.int32, device=DEV)
  def reset(self):
    self.state.fill_(NAN)
    lib = _lib()
    lib.check(lib.lib().bz_search_candidate(None, None, None, 0, self.state.data_ptr(), lib.CANDIDATE_FIRST, 0, 0, _stream()),
              "bz_search_candidate")
  def step(self, k, P, evals, words):
    lib = _lib()
    eval_status = None if words is None else self.words.data_ptr() + 4 * k
    rc = lib.lib().bz_search_step(self.parts.data_ptr() + 8 * P * k, P, self.state.data_ptr(), self.trace.data_ptr(), eval_status,
                                  self.status.data_ptr(), k, evals, _stream())
    lib.check(rc, "bz_search_step")
  def load(self, parts, words, evals):
    P = len(parts[0])
    self.parts[:evals * P].copy_(torch.tensor(parts, dtype=torch.float64).reshape(-1))
    if words is not None:
      self.words[:evals].copy_(torch.tensor(words, dtype=torch.int32))
    self.trace.fill_(-7.)
    self.status.fill_(GARBAGE_STATUS)
    return P
  def outcome(self, evals):
    torch.cuda.synchronize()
    trace = self.trace[:2 * evals + 1].cpu().tolist()
    return trace, int(self.status.item())

def _check_trace(trace, ys, xs, factor, what):
  assert [x.hex() for x in trace[0:2 * len(ys):2]] == [x.hex() for x in xs], what
  assert [y.hex() for y in trace[1:2 * len(ys):2]] == [y.hex() for y in ys], what
  assert trace[2 * len(ys)].hex() == float(factor).hex(), what

@pytest.mark.parametrize("name", [name for name, _ in line_scapes.SCAPES])
def test_transition_is_line_maximize_on_scripted_scores(name):
  scape = dict(line_scapes.SCAPES)[name]
  search = _Search()
  count = 0
  for evals in line_scapes.EVALS:
    for P in NPARTS:
      for pattern in (["plain"] if P == 1 else list(SHARES)):
        parts, ys = _script(scape, evals, P, pattern)
        xs, factor, _ = _oracle(ys)
        words, want_status = _status_words(evals, ("none", "one", "several")[count % 3])
        count += 1
        search.reset()
        search.load(parts, words, evals)
        for k in range(evals):
          search.step(k, P, evals, words)
        trace, status = search.outcome(evals)
        what = (name, evals, P, pattern)
        _check_trace(trace, ys, xs, factor, what)
        assert status == want_status, (what, words, status)

def test_the_scripts_reach_the_transitions_edges():
  """ The scripted searches above do what they are for: expansion past 2^53, long halving runs, ties,
  NaN and inf scores, fl32 rounding that ties two different sums. """
  scapes = dict(line_scapes.SCAPES)
  xs, factor, _ = _oracle(_script(scapes["increasing"], 64, 1, "plain")[1])
  assert factor == 2. ** 63 and xs[-1] > 2. ** 53
  xs, _, _ = _oracle(_script(scapes["decreasing"], 40, 1, "plain")[1])
  assert min(xs[1:]) < 1e-25                        # about 2k halvings at call k
  _, ys = _script(scapes["increasing-sub-ulp"], 8, 1, "plain")
  assert len(set(ys[1:])) == 1
  _, ys = _script(scapes["plateau"], 8, 3, "halfway")
  assert ys[0] == 1. and _fl32(1. + 2. ** -24) == 1.
  _, ys = _script(scapes["increasing"], 8, 2, "overflow-edge")
  assert ys[0] == INF and ys[1] == INF              # above FLT_MAX + ulp / 2, and exactly there (to even)
  _, ys = _script(scapes["decreasing"], 8, 2, "overflow-edge")
  assert ys[1] == FLT_MAX                           # just below
  parts, ys = _script(scapes["increasing"], 8, 3, "rank-order")
  assert ys[5] == 5. and _fl32(_sum_in_rank_order(parts[5][::-1])) == 0.

# ---------------------------------------------------------------------------- #
# K8: the candidate rows of the factors the transition leaves

def _specials(d, seed):
  """ A row of d floats holding +-0, fp32 subnormals, +-inf, NaN and +-FLT_MAX among scaled normals. """
  gen = torch.Generator().manual_seed(seed)
  values = torch.randn(d, generator=gen) * torch.pow(2., torch.randint(-30, 30, (d,), generator=gen).float())
  specials = torch.tensor([0., -0., FLT_TRUE_MIN, -FLT_TRUE_MIN, FLT_MIN / 3, INF, -INF, NAN, FLT_MAX, -FLT_MAX, 1., -FLT_MIN])
  pick = torch.randint(0, 3, (d,), generator=gen) == 0
  values[pick] = specials[torch.randint(0, len(specials), (int(pick.sum()),), generator=gen)]
  if d >= len(specials):
    values[:len(specials)] = specials
    values[-len(specials):] = specials.flip(0)
  return values

def _view(buf, offset, d):
  return buf[offset:offset + d]

def _statement(avg, att, x, negative, kind, final):
  """ The reference's candidate row (identical.py:70-72, :83-85; empire.py:54, :61). """
  if kind == "empire-strict":
    return avg.mul(-x)
  return avg + ((-x if negative and not final else x) * att)

def _bits(t):
  return t.view(torch.int32)

@pytest.mark.parametrize("d", [1, 3, 1031, 70001])
def test_candidate_rows_follow_the_transition(d):
  lib = _lib()
  search = _Search()
  count = 0
  for offsets in ((0, 0, 0), (1, 1, 1), (3, 3, 3), (1, 2, 3)):
    avg_buf = torch.empty(d + 4, device=DEV)
    att_buf = torch.empty(d + 4, device=DEV)
    avg = _view(avg_buf, offsets[0], d).copy_(_specials(d, 1 + d))
    att = _view(att_buf, offsets[1], d).copy_(_specials(d, 2 + d))
    for name in ("increasing", "increasing-x", "decreasing", "plateau", "nan-first", "edges", "random"):
      scape = dict(line_scapes.SCAPES)[name]
      for evals in (1, 2, 16, 64, 200):
        kind, negative = (("identical", False), ("identical", True), ("empire-strict", False), ("empire-strict", True))[count % 4]
        count += 1
        code = 1 if kind == "empire-strict" else 0
        parts, ys = _script(scape, evals, 1, "plain")
        xs, factor, after = _oracle(ys)
        rows = torch.full((evals + 2, d + 8), NAN, device=DEV)
        byz = [_view(rows[j], offsets[2], d) for j in range(evals + 2)]
        search.load(parts, None, evals)
        search.state.fill_(NAN)
        def candidate(which, j):
          rc = lib.lib().bz_search_candidate(avg.data_ptr(), None if code else att.data_ptr(), byz[j].data_ptr(), d,
                                             search.state.data_ptr(), which, int(negative), code, _stream())
          lib.check(rc, "bz_search_candidate")
        candidate(lib.CANDIDATE_FIRST, 0)
        for k in range(evals):
          search.step(k, 1, evals, None)
          candidate(lib.CANDIDATE_NEXT, k + 1)
        candidate(lib.CANDIDATE_FINAL, evals + 1)
        trace, _ = search.outcome(evals)
        what = (d, offsets, name, evals, kind, negative)
        _check_trace(trace, ys, xs, factor, what)
        factors = [0.] + xs[1:] + [after]                 # the x of each NEXT row: the next evaluation's
        for j, x in enumerate(factors):
          want = _statement(avg, att, x, negative, kind, False)
          assert torch.equal(_bits(byz[j]), _bits(want)), (what, j, x)
        want = _statement(avg, att, factor, negative, kind, True)
        assert torch.equal(_bits(byz[evals + 1]), _bits(want)), (what, "final", factor)

# ---------------------------------------------------------------------------- #
# Every search path on landscapes of ties and non-finite scores

EVALS = 12
BIG = 2. ** 100            # x * BIG is an outlier for every factor a 12-evaluation search tries but 0
GARS = ["average", "median", "trmean", "phocas", "meamed", "krum", "bulyan", "brute", "aksel", "cge"]
COORDINATE = ["average", "median", "trmean", "phocas", "meamed"]
WIDE = ["krum", "bulyan", "aksel", "cge"]

def _f_of(gar, n):
  from test_cuda_linesearch import F_OF
  if (gar, n) in F_OF:
    return F_OF[(gar, n)]
  if n == 64:
    return 1 if gar == "brute" else 15            # Bulyan: 4f + 3 <= n; brute: C(n, n - f) subsets
  return 24                                        # n = 100

def _rule(gar):
  import byzantinemomentum_b200 as bz
  return bz.wide_gars[gar] if gar in WIDE else bz.gars[gar]

def _landscapes(gar, honest, f):
  """ (name, kind, honest rows, avg, att) whose scores take a few levels only: exact ties (outputs that are
  the same bits), 0, NaN, +inf, and finite levels far apart:
    outlier      the candidate of any x > 0 is an outlier the rule ignores (its output stops depending on x:
                 exact ties), or averages in (average: +inf);
    zero         the same, `avg` the output on that plateau: y = 0 exactly;
    nan-at-zero  `att` is +inf: the candidate of x = 0 is 0 * inf = NaN, every other one +inf (not against
                 Aksel: a NaN median makes every distance NaN, and Aksel then averages the plateau's rows in
                 index order, the same rows summed in another order: a tie within rounding);
    overflow     `att` is FLT_MAX: x * att overflows to +inf once x > 1;
    empire-ties  empire-strict with `avg` = 0: the candidate of every x is the zero row (-0.0 for x > 0), every
                 score the same;
    empire-nan   the same with one +inf in `avg`: NaN in the candidate of x = 0, -inf in the others, and
                 every score +inf or NaN. """
  d = honest[0].numel()
  mean = torch.stack(honest).mean(dim=0)
  big = torch.full((d,), BIG, device=DEV)
  plateau = _rule(gar)(gradients=honest + [mean + big] * f, f=f)
  zero_inf = torch.zeros(d, device=DEV)
  zero_inf[d // 2] = INF
  cases = [("outlier", "identical", honest, mean, big), ("zero", "identical", honest, plateau, big),
           ("nan-at-zero", "identical", honest, mean, torch.full((d,), INF, device=DEV)),
           ("overflow", "identical", honest, mean, torch.full((d,), FLT_MAX, device=DEV)),
           ("empire-ties", "empire-strict", honest, torch.zeros(d, device=DEV), None),
           ("empire-nan", "empire-strict", honest, zero_inf, None)]
  return [case for case in cases if not (gar == "aksel" and case[0] == "nan-at-zero")]

def _cases(gar, honest, f):
  for name, kind, rows, avg, att in _landscapes(gar, honest, f):
    for negative in ((False, True) if kind == "identical" else (False,)):
      yield name, kind, negative, rows, avg, att

def _candidate(avg, att, x, negative, kind):
  """ The reference's statements (identical.py:70-72, empire.py:54): -x is -0.0 at x = 0. """
  if kind == "identical":
    return avg + (-x if negative else x) * att
  return avg.mul(-x)

def _host_search(gar, honest, f, avg, att, negative, kind):
  """ The reference's host loop (`eval_factor` in identical.py:67-77, empire.py:51-59, then `line_maximize`)
  over this library's plain rule: (xs, ys, factor).  A failed Bulyan or brute call scores NaN, as the
  device search does.  Asserts that two finite non-zero scores of outputs that are not the same bits lie
  more than 1e-5 apart (relative), so that the device's scores, summed in another order, order the same
  way, and outputs that are the same bits tie on every path. """
  from byzantinemomentum_b200 import engine
  xs, ys, outs = [], [], []
  def eval_factor(x):
    aggregated = _rule(gar)(gradients=honest + [_candidate(avg, att, x, negative, kind)] * f, f=f)
    outs.append(_bits(aggregated).clone())
    aggregated.sub_(avg)
    xs.append(x)
    ys.append(aggregated.dot(aggregated).item())
    return ys[-1]
  engine.config.strict_status = False
  try:
    factor = line_oracle.line_maximize(eval_factor, EVALS)
  finally:
    engine.config.strict_status = True
  for i in range(EVALS):
    for j in range(i):
      a, b = sorted((ys[i], ys[j]))
      if math.isfinite(a) and math.isfinite(b) and a != 0. and not torch.equal(outs[i], outs[j]):
        assert b - a > 1e-5 * b, (gar, kind, negative, xs[j], xs[i], ys[j], ys[i])
  return xs, ys, factor

_HOST = {}

def _case(gar, n):
  """ The landscapes of (gar, n) and the host loop of each, computed once: f and [(name, kind, negative,
  honest rows, avg, att, host loop)]. """
  if (gar, n) not in _HOST:
    from test_cuda_linesearch import _honest
    f = _f_of(gar, n)
    honest = _honest(n - f, 37, 1000 + n)
    _HOST[(gar, n)] = f, [(name, kind, negative, rows, avg, att, _host_search(gar, rows, f, avg, att, negative, kind))
                          for name, kind, negative, rows, avg, att in _cases(gar, honest, f)]
  return _HOST[(gar, n)]

def _outcome(record):
  host = record.cpu()
  values = host.tolist()
  return values[2 * EVALS], [(values[2 * k], values[2 * k + 1]) for k in range(EVALS)], int(host[-1:].view(torch.int32)[0])

def _check_host(record, byz, host, avg, att, negative, kind, what):
  """ The device search is the host loop: the x sequence, the factor and the Byzantine gradient bit for bit,
  every score that is not finite or is 0 bit for bit, the finite ones within 4e-6. """
  hxs, hys, hfactor = host
  factor, trace, status = _outcome(record)
  assert [x.hex() for x, _ in trace] == [x.hex() for x in hxs], (what, trace, hxs, hys)
  assert factor.hex() == float(hfactor).hex(), what
  for (x, y), hy in zip(trace, hys):
    if math.isfinite(hy) and hy != 0.:
      assert abs(y - hy) <= 4e-6 * hy, (what, x, y, hy)
    else:
      assert y.hex() == hy.hex(), (what, x, y, hy)
  assert status == 0 or any(math.isnan(y) for y in hys), (what, status)
  final = avg + factor * att if kind == "identical" else avg.mul(-factor)
  assert torch.equal(_bits(byz), _bits(final)), (what, factor)

def _check_replay(search, what):
  """ One replay of `search.graph()` rewrites the eager search's record and `byz`, bit for bit. """
  torch.cuda.synchronize()
  record, byz = search.record.clone(), search.byz.clone()
  replay = search.graph()
  search.record.fill_(-1.)
  search.byz.fill_(-1.)
  replay()
  torch.cuda.synchronize()
  assert torch.equal(search.record[:-1].view(torch.int64), record[:-1].view(torch.int64)), what
  assert torch.equal(search.record[-1:].view(torch.int32)[:1], record[-1:].view(torch.int32)[:1]), what
  assert torch.equal(_bits(search.byz), _bits(byz)), what

def _single_gpu(gar, n):
  from byzantinemomentum_b200 import engine
  f, cases = _case(gar, n)
  for i, (name, kind, negative, honest, avg, att, host) in enumerate(cases):
    search = engine.LineSearch(gar, honest, f, f, avg, att, EVALS, negative=negative, kind=kind)
    search()
    torch.cuda.synchronize()
    what = (gar, n, name, kind, negative)
    _check_host(search.record, search.byz, host, avg, att, negative, kind, what)
    if i == 2:
      _check_replay(search, what)

@pytest.mark.parametrize("n", [11, 64])
@pytest.mark.parametrize("gar", GARS)
def test_single_gpu_search_on_ties_and_non_finite_scores(gar, n):
  """ engine.LineSearch up to 64 rows (`bz_line_search`). """
  _single_gpu(gar, n)

@pytest.mark.parametrize("gar", COORDINATE + WIDE)
def test_search_at_100_rows_on_ties_and_non_finite_scores(gar):
  """ engine.LineSearch at 100 rows: the coordinate-wise rules through `bz_line_search`, Multi-Krum, Bulyan,
  Aksel and CGE through `bz_distance_line_search`. """
  _single_gpu(gar, 100)

def _sharded(gar, n, R, wide):
  from byzantinemomentum_b200 import sharded
  from test_cuda_sharded_search import _emulate
  f, cases = _case(gar, n)
  for i, (name, kind, negative, honest, avg, att, host) in enumerate(cases):
    what = (gar, n, R, wide, name, kind, negative)
    if R == 1:
      search = sharded.ShardedLineSearch(gar, honest, f, f, avg, att, EVALS, negative=negative, kind=kind, exchange="nccl", wide=wide)
      search()
      torch.cuda.synchronize()
      _check_host(search.record, search.byz, host, avg, att, negative, kind, what)
      if i == 2:
        _check_replay(search, what)
      continue
    inst, _ = _emulate(gar, honest, f, avg, att, R, False, evals=EVALS, negative=negative, kind=kind, wide=wide)
    for s in inst[1:]:
      assert torch.equal(s.record.view(torch.int64), inst[0].record.view(torch.int64)), what
    _check_host(inst[0].record, torch.cat([s.byz for s in inst]), host, avg, att, negative, kind, what)

@pytest.mark.parametrize("R", [1, 3])
@pytest.mark.parametrize("gar", GARS)
def test_sharded_search_on_ties_and_non_finite_scores(gar, R):
  """ ShardedLineSearch with the collective exchange, on one rank and on 3 ranks emulated on one GPU. """
  _sharded(gar, 11, R, False)

@pytest.mark.parametrize("R", [1, 3])
@pytest.mark.parametrize("gar", WIDE)
def test_wide_sharded_search_on_ties_and_non_finite_scores(gar, R):
  """ ShardedLineSearch(wide=True) at 100 rows, on one rank and on 3 emulated ranks. """
  _sharded(gar, 100, R, True)

@pytest.mark.parametrize("gar", GARS)
def test_fused_search_on_ties_and_non_finite_scores(gar):
  """ ShardedLineSearch(exchange="fused"): on 2 ranks emulated on one GPU (each exchange checked against the
  collective stages), and on one rank with a graph replay. """
  from byzantinemomentum_b200 import sharded
  from test_cuda_search_peers import _emulate
  f, cases = _case(gar, 11)
  for i, (name, kind, negative, honest, avg, att, host) in enumerate(cases):
    what = (gar, name, kind, negative)
    fused, _ = _emulate(gar, honest, f, avg, att, 2, evals=EVALS, searches=1, negative=negative, kind=kind)
    assert torch.equal(fused[1].record.view(torch.int64), fused[0].record.view(torch.int64)), what
    _check_host(fused[0].record, torch.cat([s.byz for s in fused]), host, avg, att, negative, kind, what)
    if i == 2:
      search = sharded.ShardedLineSearch(gar, honest, f, f, avg, att, EVALS, negative=negative, kind=kind, exchange="fused")
      search()
      torch.cuda.synchronize()
      _check_host(search.record, search.byz, host, avg, att, negative, kind, what + ("one rank",))
      _check_replay(search, what)
