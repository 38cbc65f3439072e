"""Activation-traffic model of `benchmarks/nn_bench.py --traffic` (no GPU): the backward pair of a closing batch norm moves 7
activation-sized tensors (statistics: dy, x, y read and the masked gradient written; apply: the masked gradient and x read, dx
written), one fewer than when the apply kernel masked dy again."""

import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))

import nn_bench  # noqa: E402


def test_closing_pair_counts_seven_tensors():
  workers, batch = 8, 32
  norms, _ = nn_bench.norm_layers(224)
  closing = [2 * workers * batch * math.prod(shape) for shape, _, closes in norms if closes]
  paired = [S for S in closing if S > nn_bench.FUSED_MB[1] << 20]
  sums = nn_bench.traffic(workers, batch, 224)
  count, before, after = sums["bn backward, pair, closing"]
  assert count == len(paired) == 15
  assert after == 7 * sum(paired)
  assert before == 8 * sum(paired)
  assert round(after / 1e9, 2) == 15.83


def test_other_backward_pairs_unchanged():
  sums = nn_bench.traffic(8, 32, 224)
  assert sums["bn backward, pair, no ReLU"][1] == sums["bn backward, pair, no ReLU"][2]
  count, before, after = sums["bn backward, pair, ReLU"]
  assert before * 5 == after * 7   # 7S -> 5S: y no longer read by either pass
  assert nn_bench.bn_pass(100 << 20, True, True, True) == ("bn backward, pair, closing", 8 * (100 << 20), 7 * (100 << 20))
  assert nn_bench.bn_pass(10 << 20, True, True, True)[1:] == (5 * (10 << 20), 5 * (10 << 20))   # single launch: dy, x, y, dx, masked
