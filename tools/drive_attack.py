#!/usr/bin/env python3
# coding: utf-8
"""Run the UNMODIFIED reference `attack.py` offline, with the CUDA rules registered.

The reference downloads its datasets (torchvision); here `experiments.make_datasets` — looked up
at call time by attack.py:530 — is replaced by a generator of synthetic batches of the right
shape (`experiments/dataset.py:187-190` accepts a generator), the rules of this repository are
registered through the reference's own `aggregators.register` under `b200-<name>`
(`plugin.install`), optionally the study metrics are swapped (`plugin.install_tools`) and the
line-searching attacks replaced (`plugin.install_attacks`), and `attack.py` is executed with `runpy`
exactly as `python3 attack.py <args>` would.

    python tools/drive_attack.py --reference /path/to/ByzantineMomentum --shape mnist -- \\
        --gar b200-krum --nb-workers 11 --nb-decl-byz 3 --nb-real-byz 3 --attack empire \\
        --attack-args factor:1.1 --model simples-full --nb-steps 3 --device cuda:0

Nothing in the reference is modified; no file of it is copied.
"""

import argparse
import hashlib
import pathlib
import runpy
import sys

SHAPES = {"mnist": ((1, 28, 28), 10), "cifar10": ((3, 32, 32), 10), "cifar100": ((3, 32, 32), 100)}

CLIP_AND_CLONE = """          # Gradient clip and append
          if args.gradient_clip is not None:
            grad_norm = grad.norm().item()
            if grad_norm > args.gradient_clip:
              grad.mul_(args.gradient_clip / grad_norm)
          grad_sampleds.append(grad.clone().detach_())
"""
CLIP_AND_CLONE_NEW = """          # (byzantinemomentum_b200) clip + clone + momentum placement in one pass, into a row of the stack
          grad_sampleds.append(__bz_rows.push(len(grad_sampleds), grad, args, globals()))
"""
MOMENTUM = """    if args.momentum_at == "worker":
      grad_honests = list()
      for gmtm, grad in zip(grad_momentum_workers, grad_sampleds[:args.nb_honests]):
        gmtm.mul_(args.momentum).add_(grad, alpha=(1. - args.dampening))
        grad_honests.append(gmtm)
    elif args.momentum_at == "server":
      grad_honests = list()
      for grad in grad_sampleds[:args.nb_honests]:
        grad_honests.append(grad.mul(1. - args.dampening).add_(grad_momentum_server, alpha=args.momentum))
"""
MOMENTUM_NEW = """    if args.momentum_at == "worker":
      grad_honests = __bz_rows.honests_worker(grad_momentum_workers, grad_sampleds, args)
    elif args.momentum_at == "server":
      grad_honests = __bz_rows.honests_server(grad_momentum_server, grad_sampleds, args)
"""

# The study block (attack.py:846-866) is located by the two comment lines that bracket it and checked
# by the digest of what lies between them: nothing is rewritten unless it is exactly the known text.
STUDY_BEGIN = "      # Compute the sampled and honest gradients norm average, norm deviation and max absolute coordinate\n"
STUDY_END = "      # Store the new past gradient (automatic rolling)\n"
STUDY_SHA256 = "be291ae9bc7ca4313c63ede421a64febc8c89cb15301cd16a8231a088f7d8b4f"
STUDY_NEW = """      # (byzantinemomentum_b200) the averages, norms, cosines and the curvature of this step in a handful of
      # device passes and one host read
      globals().update(__bz_rows.study(grad_sampleds, grad_honests, grad_attacks, grad_defense, grad_pasts, args))
"""

class FusedRows:
  """ What the rewritten statements call.  CUDA gradients go through `GradientStack.push` (one
  kernel per worker); anything else runs the reference's own statements, unchanged. """
  def __init__(self, bz, torch):
    self.bz, self.torch, self.stack, self.fused = bz, torch, None, False
    self.pushes = 0
    self.studies = 0
  def study(self, sampleds, honests, attacks, defense, pasts, args):
    """ attack.py:846-866 -> engine.study_step (CUDA gradients only: the product has no CPU path). """
    if not defense.is_cuda:
      raise SystemExit("drive_attack --fuse-study: the study step runs on CUDA gradients only (use --device cuda:N)")
    self.studies += 1
    out = self.bz.engine.study_step(sampleds, honests, attacks, defense, [(p.grad, p.norm) for p in pasts], args.momentum)
    out["defense_grad"] = defense
    return out
  def push(self, i, grad, args, g):
    if not grad.is_cuda:
      self.fused = False
      if args.gradient_clip is not None:
        grad_norm = grad.norm().item()
        if grad_norm > args.gradient_clip:
          grad.mul_(args.gradient_clip / grad_norm)
      return grad.clone().detach_()
    n = max(args.nb_honests, args.nb_for_study)
    if self.stack is None or self.stack.n != n or self.stack.d != grad.numel() or self.stack.device != grad.device:
      self.stack = self.bz.GradientStack(n, grad.numel(), grad.device)
    self.fused = True
    self.pushes += 1
    kwargs = {}
    if i < args.nb_honests:
      if args.momentum_at == "worker":
        kwargs = dict(worker_momentum=g["grad_momentum_workers"][i], mu=args.momentum, dampening=args.dampening)
      elif args.momentum_at == "server":
        kwargs = dict(server_momentum=g["grad_momentum_server"], mu=args.momentum, dampening=args.dampening)
    return self.stack.push(i, grad.detach(), clip=args.gradient_clip, **kwargs)
  def honests_worker(self, workers, sampleds, args):
    if self.fused:
      return list(workers[:args.nb_honests])                  # already updated by push
    out = list()
    for gmtm, grad in zip(workers, sampleds[:args.nb_honests]):
      gmtm.mul_(args.momentum).add_(grad, alpha=(1. - args.dampening))
      out.append(gmtm)
    return out
  def honests_server(self, server, sampleds, args):
    if self.fused:
      return self.stack.honest(args.nb_honests)
    return [grad.mul(1. - args.dampening).add_(server, alpha=args.momentum) for grad in sampleds[:args.nb_honests]]

def rewrite(source, fuse, fuse_study):
  """ The source of attack.py with the statement groups above swapped.  Each anchor must occur exactly
  as often as in the reference (2 and 1; the study block once, with the known digest), else SystemExit. """
  if fuse:
    if source.count(CLIP_AND_CLONE) != 2 or source.count(MOMENTUM) != 1:
      raise SystemExit("drive_attack: attack.py does not contain the expected statements; refusing to rewrite")
    source = source.replace(CLIP_AND_CLONE, CLIP_AND_CLONE_NEW).replace(MOMENTUM, MOMENTUM_NEW)
  if fuse_study:
    if source.count(STUDY_BEGIN) != 1 or source.count(STUDY_END) != 1:
      raise SystemExit("drive_attack: attack.py does not contain the expected study block; refusing to rewrite")
    lo, hi = source.index(STUDY_BEGIN), source.index(STUDY_END)
    if lo >= hi or hashlib.sha256(source[lo:hi].encode()).hexdigest() != STUDY_SHA256:
      raise SystemExit("drive_attack: the study block of attack.py is not the known one; refusing to rewrite")
    source = source[:lo] + STUDY_NEW + source[hi:]
  return source

def run_attack(path, fuse, helper, fuse_study=False):
  """ `python3 attack.py` (sys.argv already set): plain runpy, or — with `fuse` / `fuse_study` — the
  same source with the statement groups above swapped in memory (`rewrite`). """
  if not fuse and not fuse_study:
    return runpy.run_path(str(path), run_name="__main__")
  source = rewrite(path.read_text(), fuse, fuse_study)
  scope = {"__name__": "__main__", "__file__": str(path), "__builtins__": __builtins__, "__bz_rows": helper}
  exec(compile(source, str(path), "exec"), scope)
  return scope

def find_reference(root):
  """ $BYZ_REFERENCE when it holds attack.py. """
  import os
  places = ([pathlib.Path(os.environ["BYZ_REFERENCE"])] if os.environ.get("BYZ_REFERENCE") else [])
  for path in places:
    if (path / "aggregators" / "__init__.py").exists() and (path / "attack.py").exists():
      return path.resolve()
  return None

def main():
  parser = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  parser.add_argument("--reference", default=None, help="root of the ByzantineMomentum checkout (default: $BYZ_REFERENCE)")
  parser.add_argument("--count-calls", action="store_true", help="count the calls of every registered rule and its influence(); print `gar-calls <tag> <name> <calls> <influence calls>` lines after each run")
  parser.add_argument("--shape", default="mnist", choices=sorted(SHAPES), help="shape of the synthetic samples")
  parser.add_argument("--override", action="store_true", help="replace the stock rules instead of adding b200-<name>")
  parser.add_argument("--install-tools", action="store_true", help="also swap tools.compute_avg_dev_max for CUDA samples")
  parser.add_argument("--fuse-gradients", action="store_true",
    help="execute attack.py with its per-worker clip/clone/momentum statements (attack.py:775-780, 790-795, 799-808) replaced IN MEMORY by GradientStack.push (the file on disk is not touched; every anchor must match exactly)")
  parser.add_argument("--fuse-study", action="store_true",
    help="execute attack.py with its study block (attack.py:846-866: three compute_avg_dev_max, the defense norm, six cosines, the past cosine and the curvature: 9 + nb_for_study_past host syncs) replaced IN MEMORY by engine.study_step (one host read for all dot products)")
  parser.add_argument("--fuse-attacks", action="store_true",
    help="replace the little, empire, bulyan and empire-strict attacks (plugin.install_attacks): with a negative factor against a b200 rule, the whole line search (attacks/identical.py:67-77: 16 rule calls and 16 host syncs per step by default) runs on the device with one host read")
  parser.add_argument("--batch", default=None, help="JSON file with a list of {tag, args}: run attack.py once per entry in this process")
  parser.add_argument("rest", nargs=argparse.REMAINDER, help="arguments of attack.py (after --)")
  args = parser.parse_args()
  rest = args.rest[1:] if args.rest[:1] == ["--"] else args.rest
  root = pathlib.Path(__file__).resolve().parent.parent
  sys.path.insert(0, str(root))
  if args.reference is None:
    ref = find_reference(root)
    if ref is None:
      raise SystemExit("no reference found (set $BYZ_REFERENCE or pass --reference)")
  else:
    ref = pathlib.Path(args.reference).resolve()
  sys.path.insert(0, str(ref))

  import torch
  import aggregators
  import attacks
  import experiments
  import tools
  import byzantinemomentum_b200 as bz

  def make_datasets(dataset, train_batch, test_batch, **kwargs):
    # the shape follows attack.py's --dataset when it names a known one, else --shape
    sample_shape, classes = SHAPES.get(str(dataset).lower(), SHAPES[args.shape])
    def batches(size, seed):
      gen = torch.Generator().manual_seed(seed)
      while True:
        yield torch.randn((size,) + sample_shape, generator=gen), torch.randint(classes, (size,), generator=gen)
    return experiments.Dataset(batches(train_batch or 32, 1), name="synthetic-train"), \
           experiments.Dataset(batches(test_batch or 32, 2), name="synthetic-test")
  experiments.make_datasets = make_datasets

  names = bz.plugin.install(aggregators, override=args.override)
  stock_study = tools.compute_avg_dev_max
  if args.install_tools:
    bz.plugin.install_tools(tools)
  cuda_study = tools.compute_avg_dev_max
  if args.fuse_attacks:
    names += [f"attack {name}" for name in bz.plugin.install_attacks(attacks)]
  print(f"registered: {', '.join(names)}", flush=True)
  counts = {}
  if args.count_calls:
    def counted(fn, slot, key):
      def wrapper(*a, **kw):
        counts[key][slot] += 1
        return fn(*a, **kw)
      return wrapper
    for key, rule in list(aggregators.gars.items()):
      counts[key] = [0, 0]
      # attack.py:468 fetched nothing yet: rebuild the entry around counting closures with the
      # reference's own make_gar (aggregators/__init__.py:42-69)
      wrapped = aggregators.make_gar(counted(rule.unchecked, 0, key), rule.check, upper_bound=rule.upper_bound,
                                     influence=None if rule.influence is None else counted(rule.influence, 1, key))
      aggregators.gars[key] = wrapped
  stream = sys.__stdout__
  def report(tag):
    for key, pair in counts.items():
      if pair[0] or pair[1]:
        stream.write(f"gar-calls {tag} {key} {pair[0]} {pair[1]}\n")
      pair[0] = pair[1] = 0
    stream.flush()
  if args.batch:
    # several attack.py runs in ONE process (one interpreter start, one CUDA context)
    import json, traceback
    for job in json.loads(pathlib.Path(args.batch).read_text()):
      sys.argv = [str(ref / "attack.py")] + list(job["args"])
      tools.compute_avg_dev_max = cuda_study if job.get("install_tools", True) else stock_study
      try:
        helper = FusedRows(bz, torch)
        run_attack(ref / "attack.py", bool(job.get("fuse_gradients", args.fuse_gradients)), helper, bool(job.get("fuse_study", args.fuse_study)))
        stream.write(f"run-ok {job['tag']}\n")
        if helper.pushes:
          stream.write(f"fused-pushes {job['tag']} {helper.pushes}\n")
        if helper.studies:
          stream.write(f"fused-studies {job['tag']} {helper.studies}\n")
      except BaseException as err:      # attack.py reports fatal errors through exit(1)
        stream.write(f"run-failed {job['tag']} {type(err).__name__}: {err}\n")
        traceback.print_exc(file=stream)
      report(job["tag"])
    return
  sys.argv = [str(ref / "attack.py")] + rest
  helper = FusedRows(bz, torch)
  try:
    run_attack(ref / "attack.py", args.fuse_gradients, helper, args.fuse_study)
  finally:
    report("run")
    if helper.pushes:
      stream.write(f"fused-pushes run {helper.pushes}\n")
    if helper.studies:
      stream.write(f"fused-studies run {helper.studies}\n")

if __name__ == "__main__":
  main()
