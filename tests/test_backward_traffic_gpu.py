"""The backward pass of a residual unit with less activation traffic gives the same bits as the separate passes it replaces:
the shortcut gradient summed in the epilogue of the residual branch's first data gradient, the strided shortcut gradient added
in place at the sampled pixels, and the ReLU mask of a batch norm recomputed from its input by the statistics + apply pair."""

import pytest
import torch

pytestmark = pytest.mark.gpu


def _bits(t):
  """Bit pattern of a bf16 / fp32 tensor: NaN equals NaN, -0 differs from +0."""
  return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


@pytest.fixture
def native():
  from aggregathor_b200.ops import nn_native
  yield nn_native
  nn_native.set_gemm_epilogue("staged")
  nn_native.set_bn_fused(True)
  nn_native.set_bn_fused_limits()
  nn_native.set_deterministic(False)


@pytest.mark.parametrize("epilogue", ["staged", "regs"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("m,k,n", [(200, 64, 64), (1000, 128, 256), (777, 256, 1024), (4100, 512, 2048), (300, 64, 200)])
def test_dgrad_addend_equals_separate_add(native, epilogue, dtype, m, k, n):
  native.set_gemm_epilogue(epilogue)
  gen = torch.Generator(device="cuda").manual_seed(m + n)
  dy = torch.randn((m, k), device="cuda", generator=gen).to(dtype)
  w = (torch.randn((k, n), device="cuda", generator=gen) / k ** 0.5).to(dtype)
  addend = torch.randn((m, n), device="cuda", generator=gen).to(dtype)
  addend[0, :8] = torch.tensor([0.0, -0.0, float("inf"), float("-inf"), float("nan"), 1e-40, -1e30, 3.0])
  separate = native.add_relu_forward(addend, native.mm_nn(dy, w), False)
  summed = native.mm_nn(dy, w, addend=addend)
  torch.cuda.synchronize()
  assert torch.equal(_bits(summed), _bits(separate))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("n,c,h,w", [(4, 256, 56, 56), (2, 64, 7, 9), (3, 512, 28, 28)])
def test_subsample_accumulate_equals_scatter_and_add(native, dtype, n, c, h, w):
  gen = torch.Generator(device="cuda").manual_seed(c + h)
  dx = torch.randn((n, c, h, w), device="cuda", generator=gen).to(dtype).contiguous(memory_format=torch.channels_last)
  dx[0, :, 1, 1] = -0.0   # skipped pixel: the separate add makes it +0, the in-place one keeps -0 (equal under torch.equal)
  dy = torch.randn((n, c, -(-h // 2), -(-w // 2)), device="cuda", generator=gen).to(dtype).contiguous(memory_format=torch.channels_last)
  separate = native.add_relu_forward(native.subsample_backward(dy, dx.shape, 2), dx, False)
  summed = native.subsample_accumulate(dx.clone(), dy, 2)
  torch.cuda.synchronize()
  assert torch.equal(summed, separate)
  assert torch.equal(summed.abs(), separate.abs())
  assert torch.signbit(summed[0, :, 1, 1]).all()


def _planted(groups, rows_per_group, c, dtype, gen):
  x = (torch.randn((groups * rows_per_group, c), device="cuda", generator=gen) * 2 + 0.5).to(dtype)
  x[3, 0] = float("nan")
  x[5, 1] = float("inf")
  x[7, 2] = float("-inf")
  x[::3, 3] = -0.0
  x[::5, 4] = 0.0
  gamma = torch.rand(c, device="cuda", generator=gen) + 0.5
  beta = torch.randn(c, device="cuda", generator=gen) * 0.1
  gamma[5], beta[5] = 3e-41, 0.0   # fma(x, scale, shift) is a tiny denormal: some round to 0 in bf16, some do not
  gamma[6], beta[6] = 1e-38, 0.0
  return x, gamma, beta


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("forward", ["fused", "pair"])
@pytest.mark.parametrize("groups", [1, 8])
def test_recomputed_mask_equals_stored_mask(native, dtype, forward, groups):
  if forward == "fused" and dtype == torch.float32:
    pytest.skip("the single-launch forward is bf16 only")
  c, rows_per_group = 128, 1024
  gen = torch.Generator(device="cuda").manual_seed(groups)
  x2d, gamma, beta = _planted(groups, rows_per_group, c, dtype, gen)
  x = x2d.view(groups * rows_per_group, 1, 1, c).permute(0, 3, 1, 2)
  dy = torch.randn_like(x2d, dtype=torch.float32).to(dtype).view(x.shape[0], 1, 1, c).permute(0, 3, 1, 2)
  moving_mean, moving_var = torch.zeros(c, device="cuda"), torch.ones(c, device="cuda")
  native.set_bn_fused(forward == "fused")
  native.set_bn_fused_limits(min_rows=1)
  y, mean, rstd, coef = native.batchnorm_forward(x, gamma, beta, moving_mean, moving_var, 0.9, 1e-5, True, groups, coef=True)
  assert ((y > 0) == (native.batchnorm_forward(x, gamma, beta, moving_mean, moving_var, 0.9, 1e-5, True, groups)[0] > 0)).all()
  assert (y[:, 5] == 0).any() and (y[:, 5] > 0).any()
  native.set_bn_fused(False)   # the pair backward: the path that recomputes the mask
  outs = []
  for mask_coef in (None, coef):
    dgamma, dbeta = torch.zeros((groups, c), device="cuda"), torch.zeros((groups, c), device="cuda")
    dx = native.batchnorm_backward(dy, x, y, gamma, mean, rstd, True, dgamma[0], dbeta[0], groups, c, mask_coef=mask_coef)
    outs.append((dx, dgamma, dbeta))
  torch.cuda.synchronize()
  for stored, recomputed in zip(*outs):
    assert torch.equal(_bits(recomputed), _bits(stored))


def test_batched_resnet_step_matches_separate_passes(native, monkeypatch):
  """A batched slim resnet_v1_50 step at 64 x 64 through the pair batch norm and the staged epilogue: every worker's gradient row is
  the same, bit for bit, as with the shortcut gradients added by separate passes and the ReLU masks read from y."""
  from aggregathor_b200.engine.flat import FlatLayout
  from aggregathor_b200.models import Context, core, nets_factory
  from aggregathor_b200.ops import nn as nn_ops
  groups, batch = 4, 8
  model = nets_factory.get_network("resnet_v1_50", 1000)
  layout, states = FlatLayout(), {}
  model.declare(layout, states)
  layout.freeze()
  host = torch.zeros(layout.padded_size)
  host_states = {k: torch.zeros(v) for k, v in states.items()}
  model.initialize(layout.views(host), host_states, torch.Generator().manual_seed(1))
  params = host.cuda()
  gen = torch.Generator(device="cuda").manual_seed(3)
  x = torch.randn((groups * batch, 3, 64, 64), device="cuda", generator=gen).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
  labels = torch.randint(0, 1000, (groups * batch,), device="cuda", generator=gen)

  def step():
    ctx = Context("native", True, torch.bfloat16, "cuda")
    ctx.groups, ctx.group_stride = groups, layout.padded_size
    ctx.master = layout.views(params)
    ctx.weights = layout.views(params.to(torch.bfloat16))
    ctx.state = {k: v.cuda() for k, v in host_states.items()}
    grads = torch.zeros((groups, layout.padded_size), device="cuda")
    ctx.grads = layout.views(grads[0])
    loss = model.loss_and_backward(x, labels, ctx)
    torch.cuda.synchronize()
    return loss.clone(), grads

  native.set_deterministic(True)
  native.set_bn_fused(False)
  calls = {"summed": 0, "recomputed": 0}
  summed_backward, batchnorm_backward = core.Residual._backward_summed, native.batchnorm_backward

  def counting_summed(self, db, dy, ctx):
    calls["summed"] += 1
    return summed_backward(self, db, dy, ctx)

  def counting_batchnorm(*args, mask_coef=None, **kwargs):
    calls["recomputed"] += mask_coef is not None
    return batchnorm_backward(*args, mask_coef=mask_coef, **kwargs)

  monkeypatch.setattr(core.Residual, "_backward_summed", counting_summed)
  monkeypatch.setattr(native, "batchnorm_backward", counting_batchnorm)
  loss, grads = step()
  assert calls["summed"] == 16 and calls["recomputed"] > 0

  def separate(self, db, dy, ctx):
    for layer in reversed(self.residual.layers[:-1]):
      db = layer.backward(db, ctx)
    return nn_ops.add_forward(ctx.backend, self.shortcut.backward(dy, ctx), db)

  monkeypatch.setattr(core.Residual, "_backward_summed", separate)
  monkeypatch.setattr(native, "batchnorm_backward", lambda *args, mask_coef=None, **kwargs: batchnorm_backward(*args, **kwargs))
  ref_loss, ref_grads = step()
  torch.testing.assert_close(loss, ref_loss, rtol=1e-5, atol=0)   # the per-worker loss is summed by fp32 atomics in varying order
  assert torch.isfinite(grads).all()
  for g in range(groups):
    assert torch.equal(grads[g], ref_grads[g]), g
