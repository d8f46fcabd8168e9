# coding: utf-8
"""GPU parity pinned to the REFERENCE ITSELF at BASELINE.json's full sizes.

The goldens stop at d = 4,099 and `tests/test_cuda_fullsize.py` checks against the C oracle (a
restatement).  Here the CUDA rules are compared with what the unmodified reference returned —
`aggregators.gars[g].unchecked(gradients=<cpu rows>, f=f)` — on the SAME seeded rows, recorded
in `tests/golden/fullsize_reference.npz` by `tests/golden/make_fullsize_golden.py` (the rows
are regenerated here from torch's CPU generator by the same function):
  * bit-exact bars: the digest of the whole CUDA output must equal the digest of the
    reference's (selections are compared through what they determine: `influence()` (exact)
    and the ordered-subset mean itself, bit-exact when and only when the same rows were picked
    in the same order: krum, brute, aksel, cge);
  * tolerance bars (`tests/parity.py`: ATen tail columns, 1e-6 closest-m means): on the stored
    seeded sample of columns and the trailing `d mod 32` columns.
Sizes: C1 (median n=11 d=79,510), C2 (trmean n=25 f=10 d=1,310,922), C3 (Multi-Krum + Bulyan
n=25 f=5 d=1,310,922, empire), C5 (brute n=11 f=3 d=1,310,922), plus one C4 shard (n=51 f=12,
d=4,568,372 = 36,546,980 / 8).
"""

import numpy as np
import pytest

import conftest
import parity

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
DEV = "cuda:0"

import sys  # noqa: E402
sys.path.insert(0, str(conftest.GOLDEN_DIR))
import make_fullsize_golden as fixture  # noqa: E402

@pytest.fixture(scope="module")
def ref():
  data = np.load(fixture.OUT, allow_pickle=False)
  return {k: data[k] for k in data.files}

def _stack(ref, case, n, nb, d, seed, dist="empire"):
  """ The generator's CPU rows and their copies on the device (aliased Byzantine rows stay one
  object on both sides).  The rows must be the ones the fixture was recorded on: torch's CPU
  generator and ATen's `mean(dim=0)` (the Byzantine row) could differ on another host. """
  cpu, nh = fixture.stack(n, nb, d, seed, dist)
  assert fixture.digest(torch.stack(cpu).numpy()) == str(ref[case + "/inputs_sha256"]), \
    f"{case}: this host regenerates other input rows than the ones the reference outputs were recorded on"
  dev = [r.to(DEV) for r in cpu[:nh]]
  if nb:
    dev += [cpu[nh].to(DEV)] * nb
  return cpu, dev, nh

def _np(t):
  return t.detach().cpu().numpy()

def _key(case, rule, **kwargs):
  return fixture.key(case, rule, kwargs)

def _cols(d):
  return fixture.columns(d)

def assert_same_as_reference(got, ref, key, what):
  """ Bit-exact bar on the whole output: equal digests; on a mismatch, the stored sample says where. """
  if fixture.digest(got) != str(ref[key + "/sha256"]):
    cols = _cols(got.shape[0])
    parity.assert_bit_exact(got[cols], ref[key + "/sample"], what + " [sampled columns]")
    raise AssertionError(f"{what}: output differs from the reference outside the stored sample")

def test_c1_median(ref):
  import byzantinemomentum_b200 as bz
  for dist in ("iid", "empire"):
    cpu, dev, nh = _stack(ref, f"c1/{dist}", 11, 0 if dist == "iid" else 5, 79_510, 11, dist)
    assert_same_as_reference(_np(bz.gars["median"](gradients=dev, f=5)), ref, _key(f"c1/{dist}", "median"), f"C1 median {dist}")

def test_c2_trmean_phocas_meamed(ref):
  import byzantinemomentum_b200 as bz
  n, f, d = 25, 10, 1_310_922
  cols = _cols(d)
  body = d - d % 32
  for dist, nb in (("iid", 0), ("empire", 10)):
    cpu, dev, nh = _stack(ref, f"c2/{dist}", n, nb, d, 12, dist)
    x = np.stack([_np(r[cols]) for r in cpu])
    got = _np(bz.gars["trmean"](gradients=dev, f=f))
    k = _key(f"c2/{dist}", "trmean")
    assert fixture.digest(got[:body]) == str(ref[k + "/sha256_body"]), f"C2 trmean {dist}: body differs from the reference"
    want = ref[k + "/sample"]
    parity.assert_trmean(got[cols], want, x, f"C2 trmean {dist} [sampled columns]")   # the sample's last d mod 32 are the tail
    assert_same_as_reference(_np(bz.gars["median"](gradients=dev, f=f)), ref, _key(f"c2/{dist}", "median"), f"C2 median {dist}")
    med = ref[_key(f"c2/{dist}", "median") + "/sample"]
    for name, center in (("phocas", want), ("meamed", med)):
      theirs = ref[_key(f"c2/{dist}", name) + "/sample"]
      amb = parity.closest_ambiguous(x, n - f, center)
      parity.assert_close_scaled(_np(bz.gars[name](gradients=dev, f=f))[cols], theirs, parity.column_scale(x), f"C2 {name} {dist}", exempt=amb)
    assert_same_as_reference(_np(bz.gars["average"](gradients=dev, f=f)), ref, _key(f"c2/{dist}", "average"), f"C2 average {dist}")

def test_c3_krum_bulyan_and_the_other_distance_rules(ref):
  import byzantinemomentum_b200 as bz
  n, nb, f, d = 25, 5, 5, 1_310_922
  cols = _cols(d)
  for dist, nbyz in (("empire", nb), ("iid", 0)):
    cpu, dev, nh = _stack(ref, f"c3/{dist}", n, nbyz, d, 13, dist)
    x = np.stack([_np(r[cols]) for r in cpu])
    for name, kwargs in (("krum", {}), ("krum", dict(m=1)), ("aksel", {}), ("aksel", dict(mode="n-f")), ("cge", {})):
      k = _key(f"c3/{dist}", name, **kwargs)
      got = _np(bz.gars[name](gradients=dev, f=f, **kwargs))
      if name == "aksel":
        # aksel.py:41: distances are an fp32 ATen sum whose order depends on the thread count; the
        # selection is compared through influence below and the mean to 1e-6 (it is bit-exact
        # when the selection agrees — asserted too, on these seeds it does)
        parity.assert_close_scaled(got[cols], ref[k + "/sample"], parity.column_scale(x), f"C3 {name} {kwargs} {dist}")
      assert_same_as_reference(got, ref, k, f"C3 {name} {kwargs} {dist}")
      if nbyz:
        assert bz.gars[name].influence(dev[:nh], dev[nh:], f=f, **kwargs) == float(ref[k + "/influence"]), (name, kwargs)
    want = ref[_key(f"c3/{dist}", "bulyan") + "/sample"].astype(np.float64)
    got = _np(bz.gars["bulyan"](gradients=dev, f=f))[cols]
    # stage 2 is a closest-beta mean in topk's unspecified order: 1e-6 of the summed magnitude
    # (a different stage-1 selection would move whole coordinates by O(1)).  Coordinates with an
    # exact key tie across the closest-beta boundary have two valid answers: they are identified
    # by redoing stages 1-2 with the oracle on exactly those columns.
    scale = parity.column_scale(x)
    off = np.abs(got.astype(np.float64) - want) > 2e-6 * np.maximum(np.abs(want), scale)
    exempt = np.zeros(cols.size, dtype=bool)
    if off.any():
      bad = np.flatnonzero(off)
      assert bad.size <= 50, f"C3 bulyan {dist}: {bad.size} coordinates differ"
      from oracle import byzoracle as orc, corc
      host = [_np(r) for r in cpu]
      D = corc.pairwise_distances(host)
      border, _ = orc.bulyan_order(D, f, n - f - 2)
      stage1 = orc.bulyan_stage1(orc.as_matrix([h[cols[bad]] for h in host]), border, f, n - f - 2)
      _, amb = orc.closest_mean(stage1, stage1.shape[0] - 2 * f, orc.median(stage1), return_info=True)
      exempt[bad] = amb
    parity.assert_close_scaled(got, want, scale, f"C3 bulyan {dist}", rtol=2e-6, exempt=exempt)

def test_c5_brute(ref):
  import byzantinemomentum_b200 as bz
  n, f, d = 11, 3, 1_310_922
  for dist, nb in (("empire", 3), ("iid", 0)):
    cpu, dev, nh = _stack(ref, f"c5/{dist}", n, nb, d, 15, dist)
    k = _key(f"c5/{dist}", "brute")
    assert_same_as_reference(_np(bz.gars["brute"](gradients=dev, f=f)), ref, k, f"C5 brute {dist}")
    if nb:
      assert bz.gars["brute"].influence(dev[:nh], dev[nh:], f=f) == float(ref[k + "/influence"])

def test_c4_shard_median_trmean_n51(ref):
  import byzantinemomentum_b200 as bz
  n, f, d = 51, 12, 36_546_980 // 8
  cols = _cols(d)
  body = d - d % 32
  cpu, dev, nh = _stack(ref, "c4/empire", n, 12, d, 14, "empire")
  x = np.stack([_np(r[cols]) for r in cpu])
  k = _key("c4/empire", "trmean")
  got = _np(bz.gars["trmean"](gradients=dev, f=f))
  assert fixture.digest(got[:body]) == str(ref[k + "/sha256_body"]), "C4 shard trmean: body differs from the reference"
  parity.assert_trmean(got[cols], ref[k + "/sample"], x, "C4 shard trmean [sampled columns]")
  assert_same_as_reference(_np(bz.gars["median"](gradients=dev, f=f)), ref, _key("c4/empire", "median"), "C4 shard median")
