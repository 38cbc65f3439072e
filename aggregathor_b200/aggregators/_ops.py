"""Back-ends shared by the GAR plug-ins.

Three interchangeable implementations of every rule, mirroring the reference's
`-py` / `-tf` / `-co` triplets (`aggregators/krum.py:45-169`, `bulyan.py:43-94`):

* `host_*`   — the C++ host library `native/py_gars` through ctypes (the `-py` flavour;
               GPU tensors take a device->host->device round trip, as `tf.py_func` did);
* `torch_*`  — plain torch ops, device agnostic (the `-tf` flavour; also the fp32 test oracle);
* `cuda_*`   — the stand-alone sm_90a kernels of `native/op_gar` (the `-co` flavour).

Ordering convention everywhere: finite ascending, then non-finite; ties -> lower worker index.
"""

import ctypes
import itertools
import math

import numpy as np
import torch

from .. import tools

# ---------------------------------------------------------------------------- #
# Helpers

def stack(gradients):
  """List of n flat tensors (or an [n, d] tensor) -> contiguous [n, d] tensor."""
  if isinstance(gradients, torch.Tensor):
    if gradients.dim() != 2:
      raise tools.UserException("Expected an [n, d] tensor of gradients, got shape " + repr(tuple(gradients.shape)))
    return gradients.contiguous()
  if len(gradients) == 0:
    raise tools.UserException("Empty list of gradient to aggregate")
  return torch.stack([g.reshape(-1) for g in gradients], dim=0)


def check_krum(n, f, m=None):
  if n - f - 2 < 1:
    raise tools.UserException("Multi-Krum needs n - f - 2 >= 1 (got n = %d, f = %d)" % (n, f))
  if m is not None and not 1 <= m <= n:
    raise tools.UserException("Multi-Krum needs 1 <= m <= n (got m = %d, n = %d)" % (m, n))


def check_bulyan(n, f, m=None):
  if n < 4 * f + 3:
    raise tools.UserException("Bulyan needs n >= 4 f + 3 (got n = %d, f = %d): beta = n - 4 f - 2 must be >= 1" % (n, f))
  theta = n - 2 * f - 2
  if m is not None and not theta <= m <= n:
    raise tools.UserException("Bulyan needs n - 2 f - 2 <= m <= n (got m = %d)" % m)


def check_trimmed_mean(n, f):
  if not 0 <= 2 * f < n:
    raise tools.UserException("The trimmed mean needs 0 <= 2 f < n (got n = %d, f = %d)" % (n, f))


MDA_MAX_SETS = 1 << 20


def check_mda(n, f):
  if not 0 <= 2 * f < n:
    raise tools.UserException("MDA needs 0 <= 2 f < n (got n = %d, f = %d)" % (n, f))
  if math.comb(n, f) > MDA_MAX_SETS:
    raise tools.UserException("MDA enumerates the C(n, f) subsets of removed workers: C(%d, %d) = %d is above the bound 2^20" % (n, f, math.comb(n, f)))


GEOMETRIC_MEDIAN_MAX_ITERATIONS = 16


def check_geometric_median(n, f, iterations, nu):
  """Validate the geometric median's parameters -> (iterations, nu rounded once to fp32). `f` is not used by the algorithm; its
  breakdown point 1/2 still requires 0 <= 2 f < n."""
  if not 0 <= 2 * f < n:
    raise tools.UserException("The geometric median needs 0 <= 2 f < n (got n = %d, f = %d)" % (n, f))
  if isinstance(iterations, bool) or int(iterations) != iterations or not 1 <= iterations <= GEOMETRIC_MEDIAN_MAX_ITERATIONS:
    raise tools.UserException("The geometric median needs 1 <= iterations <= %d (got %r)" % (GEOMETRIC_MEDIAN_MAX_ITERATIONS, iterations))
  nu32 = float(torch.tensor(float(nu), dtype=torch.float32)) if math.isfinite(float(nu)) else float(nu)
  if not (math.isfinite(nu32) and nu32 > 0):
    raise tools.UserException("The geometric median needs a finite smoothing nu > 0 in fp32 (got %r)" % (nu,))
  return int(iterations), nu32


def fp32(value):
  """`value` rounded once to fp32 (non-finite values pass through)."""
  value = float(value)
  return float(torch.tensor(value, dtype=torch.float32)) if math.isfinite(value) else value


def check_centered_clipping(n, f, iterations, tau):
  """Validate centered clipping's parameters -> (iterations, tau rounded once to fp32). `f` is not used by the algorithm; as for the
  geometric median, 0 <= 2 f < n is still required."""
  if not 0 <= 2 * f < n:
    raise tools.UserException("Centered clipping needs 0 <= 2 f < n (got n = %d, f = %d)" % (n, f))
  if isinstance(iterations, bool) or int(iterations) != iterations or not 1 <= iterations <= GEOMETRIC_MEDIAN_MAX_ITERATIONS:
    raise tools.UserException("Centered clipping needs 1 <= iterations <= %d (got %r)" % (GEOMETRIC_MEDIAN_MAX_ITERATIONS, iterations))
  tau32 = fp32(tau)
  if not (math.isfinite(tau32) and tau32 > 0):
    raise tools.UserException("Centered clipping needs a finite clipping radius tau > 0 in fp32 (got %r)" % (tau,))
  return int(iterations), tau32


def check_worker_momentum(beta, dampening):
  """Validate worker momentum's coefficients -> (beta, c = 1 - dampening), both in fp32: beta and dampening are rounded once to fp32,
  then c is computed in float64 from the rounded dampening and rounded once."""
  values = []
  for name, value in (("--worker-momentum", beta), ("--worker-momentum-dampening", dampening)):
    try:
      value = fp32(value)
    except (TypeError, ValueError):
      raise tools.UserException("%s expects a number (got %r)" % (name, value))
    if not (math.isfinite(value) and 0.0 <= value < 1.0):
      raise tools.UserException("%s must be finite, >= 0 and < 1 in fp32 (got %r)" % (name, value))
    values.append(value)
  beta32, dampening32 = values
  return beta32, fp32(1.0 - dampening32)


def _rank_key(values):
  """Sort key implementing (finite ascending, non-finite last); argsort(stable) then breaks ties by index."""
  return torch.where(torch.isfinite(values), values, torch.full_like(values, float("inf")))


# ---------------------------------------------------------------------------- #
# Host C++ back-end

_host_cache = {}


def _host(symbol, dtype):
  from .. import native
  suffix = {torch.float32: "float", torch.float64: "double"}.get(dtype)
  if suffix is None:
    raise tools.UserException("Unsupported floating point type " + repr(dtype) + " for the host GARs")
  key = symbol + "_" + suffix
  if key not in _host_cache:
    lib = native.library("py_gars")
    _host_cache[key] = getattr(lib, "agb_cpu_" + key)
  return _host_cache[key]


def _ptr(tensor):
  return ctypes.c_void_p(tensor.data_ptr())


def _host_call(symbol, G, *extra, outputs=()):
  """Run `agb_cpu_<symbol>_<type>(G, n, d, *extra, out, *outputs)` on a CPU copy of G; result on G's device."""
  Gc = G.detach().to("cpu").contiguous()
  n, d = Gc.shape
  out = torch.empty(d, dtype=Gc.dtype)
  func = _host(symbol, Gc.dtype)
  status = func(_ptr(Gc), ctypes.c_size_t(n), ctypes.c_size_t(d), *[ctypes.c_size_t(e) for e in extra], _ptr(out), *[(_ptr(o) if o is not None else None) for o in outputs])
  if status != 0:
    raise tools.UserException("Host GAR " + repr(symbol) + " rejected its arguments (n = %d, d = %d, extra = %r)" % (n, d, extra))
  return out.to(G.device)


def host_average(G):
  return _host_call("average", G)


def host_average_nan(G):
  return _host_call("average_nan", G)


def host_median(G):
  return _host_call("median", G)


def host_averaged_median(G, beta):
  return _host_call("averaged_median", G, beta)


def host_krum(G, f, m, return_selected=False):
  selected = torch.empty(m, dtype=torch.int64)
  out = _host_call("krum", G, f, m, outputs=(selected, None))
  return (out, selected) if return_selected else out


def host_bulyan(G, f, m, return_weights=False):
  n = G.shape[0]
  weights = torch.empty((n - 2 * f - 2, n), dtype=G.dtype if G.dtype in (torch.float32, torch.float64) else torch.float32)
  out = _host_call("bulyan", G, f, m, outputs=(weights,))
  return (out, weights) if return_weights else out


def host_trimmed_mean(G, f):
  check_trimmed_mean(G.shape[0], f)
  return _host_call("trimmed_mean", G, f)


def host_mda(G, f, return_selected=False):
  check_mda(G.shape[0], f)
  selected = torch.empty(G.shape[0] - f, dtype=torch.int64)
  out = _host_call("mda", G, f, outputs=(selected, None))
  return (out, selected) if return_selected else out


def host_mda_select(dist, f):
  """Selection stage of MDA on an [n, n] distance matrix -> ascending ids of the n - f kept workers."""
  dist = dist.detach().to("cpu").contiguous()
  n = dist.shape[0]
  check_mda(n, f)
  selected = torch.empty(n - f, dtype=torch.int64)
  status = _host("mda_select", dist.dtype)(_ptr(dist), ctypes.c_size_t(n), ctypes.c_size_t(f), _ptr(selected))
  if status != 0:
    raise tools.UserException("Host MDA selection rejected its arguments (n = %d, f = %d)" % (n, f))
  return selected


def host_geometric_median(G, iterations, nu, return_distances=False):
  """Host library's geometric median; `return_distances` also gives the [iterations, n] squared distances D of every iteration."""
  iterations, nu = check_geometric_median(G.shape[0], 0, iterations, nu)
  Gc = G.detach().to("cpu").contiguous()
  n, d = Gc.shape
  out = torch.empty(d, dtype=Gc.dtype)
  dist = torch.empty((iterations, n), dtype=Gc.dtype)
  status = _host("geometric_median", Gc.dtype)(_ptr(Gc), ctypes.c_size_t(n), ctypes.c_size_t(d), ctypes.c_size_t(iterations), ctypes.c_double(nu),
                                               _ptr(out), _ptr(dist))
  if status != 0:
    raise tools.UserException("Host geometric median rejected its arguments (n = %d, d = %d, iterations = %d, nu = %r)" % (n, d, iterations, nu))
  out = out.to(G.device)
  return (out, dist) if return_distances else out


def host_centered_clipping(G, iterations, tau, center, return_distances=False):
  """Host library's centered clipping from the [d] `center`, which is updated in place (v <- z_T); returns z_T, and with
  `return_distances` also the [iterations, n] squared distances D of every iteration."""
  iterations, tau = check_centered_clipping(G.shape[0], 0, iterations, tau)
  Gc = G.detach().to("cpu").contiguous()
  n, d = Gc.shape
  if center.shape != (d,) or center.dtype != Gc.dtype:
    raise tools.UserException("Centered clipping needs a [%d] center of type %s (got %s, %s)" % (d, Gc.dtype, tuple(center.shape), center.dtype))
  work = center.detach().to("cpu", copy=True).contiguous()
  dist = torch.empty((iterations, n), dtype=Gc.dtype)
  status = _host("centered_clipping", Gc.dtype)(_ptr(Gc), ctypes.c_size_t(n), ctypes.c_size_t(d), ctypes.c_size_t(iterations), ctypes.c_double(tau),
                                                _ptr(work), _ptr(dist))
  if status != 0:
    raise tools.UserException("Host centered clipping rejected its arguments (n = %d, d = %d, iterations = %d, tau = %r)" % (n, d, iterations, tau))
  center.copy_(work)
  out = work.to(G.device)
  return (out, dist) if return_distances else out


def host_pairwise_distances(G):
  Gc = G.detach().to("cpu").contiguous()
  n, d = Gc.shape
  dist = torch.empty((n, n), dtype=Gc.dtype)
  _host("pairwise_distances", Gc.dtype)(_ptr(Gc), ctypes.c_size_t(n), ctypes.c_size_t(d), _ptr(dist))
  return dist


def host_bulyan_weights(dist, f, m):
  """Selection stage of Bulyan on an [n, n] distance matrix -> [theta, n] weight matrix."""
  dist = dist.detach().to("cpu").contiguous()
  n = dist.shape[0]
  weights = torch.empty((n - 2 * f - 2, n), dtype=dist.dtype)
  status = _host("bulyan_weights", dist.dtype)(_ptr(dist), ctypes.c_size_t(n), ctypes.c_size_t(f), ctypes.c_size_t(m), _ptr(weights))
  if status != 0:
    raise tools.UserException("Invalid Bulyan parameters (n = %d, f = %d, m = %d)" % (n, f, m))
  return weights


def host_squared_distance(a, b):
  a = a.detach().to("cpu").contiguous().reshape(-1)
  b = b.detach().to("cpu").contiguous().reshape(-1)
  func = _host("squared_distance", a.dtype)
  func.restype = ctypes.c_float if a.dtype == torch.float32 else ctypes.c_double
  return float(func(_ptr(a), _ptr(b), ctypes.c_size_t(a.numel())))


# ---------------------------------------------------------------------------- #
# Pure torch back-end (device agnostic; the fp32 oracle of the CUDA kernels)

def torch_average(G):
  return G.sum(dim=0) / G.shape[0]


def torch_average_nan(G):
  finite = torch.isfinite(G)
  total = torch.where(finite, G, torch.zeros_like(G)).sum(dim=0)
  return total / finite.sum(dim=0).to(G.dtype)


def torch_median(G):
  n = G.shape[0]
  order = torch.argsort(_rank_key(G), dim=0, stable=True)
  return torch.gather(G, 0, order[n // 2:n // 2 + 1]).squeeze(0)


def torch_averaged_median(G, beta):
  n = G.shape[0]
  zero = torch_median(G)
  dev = (G - zero.unsqueeze(0)).abs()
  order = torch.argsort(_rank_key(dev), dim=0, stable=True)[:beta]
  keep = torch.zeros_like(G, dtype=torch.bool).scatter_(0, order, True)
  return torch.where(keep, G, torch.zeros_like(G)).sum(dim=0) / beta


def torch_trimmed_mean(G, f):
  """Per coordinate, mean of the values ranked [f, n - f) under the ordering convention."""
  n = G.shape[0]
  check_trimmed_mean(n, f)
  order = torch.argsort(_rank_key(G), dim=0, stable=True)
  keep = torch.zeros_like(G, dtype=torch.bool).scatter_(0, order[f:n - f], True)
  return torch.where(keep, G, torch.zeros_like(G)).sum(dim=0) / (n - 2 * f)


def mda_select(dist, f, chunk=1 << 22):
  """[n, n] distances -> ascending ids of the n - f kept workers of minimum diameter; ties -> lexicographically smallest id list.
  Enumerates the kept sets in lexicographic order (`itertools.combinations`); `argmin` returns the first minimum."""
  n = dist.shape[0]
  check_mda(n, f)
  D = torch.where(torch.isfinite(dist), dist, torch.full_like(dist, float("inf")))
  size = n - f
  if size < 2:
    return torch.arange(size, dtype=torch.int64)
  sets = torch.tensor(list(itertools.combinations(range(n), size)), dtype=torch.int64, device=dist.device)
  rows = max(1, chunk // (size * size))
  diam = torch.cat([D[part[:, :, None], part[:, None, :]].amax(dim=(1, 2)) for part in sets.split(rows)])
  return sets[int(torch.argmin(diam))].cpu()


def torch_mda(G, f, return_selected=False):
  n = G.shape[0]
  check_mda(n, f)
  selected = mda_select(torch_pairwise_distances(G), f)
  out = G[selected.to(G.device)].sum(dim=0) / (n - f)
  return (out, selected) if return_selected else out


def torch_geometric_median(G, iterations, nu, return_distances=False):
  """Smoothed Weiszfeld iterations from the coordinate-wise median, in G's dtype (double inputs, more than 32 workers on a device):
  rows with a non-finite squared distance are skipped, beta_i = 1 / max(nu, sqrt(D_i)), z = (sum beta_i x_i) / (sum beta_i) with
  both sums over the kept rows in ascending order; no kept row keeps z."""
  iterations, nu = check_geometric_median(G.shape[0], 0, iterations, nu)
  n = G.shape[0]
  scalar = lambda value: torch.tensor(value, dtype=G.dtype, device=G.device)
  one, smooth = scalar(1.0), scalar(nu)
  z = torch_median(G)
  dists = []
  for _ in range(iterations):
    delta = G - z.unsqueeze(0)
    D = (delta * delta).sum(dim=1)
    dists.append(D)
    kept = [i for i in range(n) if math.isfinite(float(D[i]))]
    if not kept:
      continue
    # the square root of an fp32 value taken in fp64 and rounded once is correctly rounded (torch's CPU fp32 sqrt is not always)
    root = torch.sqrt(D.double()).to(G.dtype)
    beta = one / torch.maximum(root, smooth)
    total = torch.zeros((), dtype=G.dtype, device=G.device)
    num = torch.zeros_like(z)
    for i in kept:
      total = total + beta[i]
      num = num + beta[i] * G[i]
    z = num / total
  return (z, torch.stack(dists)) if return_distances else z


def torch_centered_clipping(G, iterations, tau, center, return_distances=False):
  """Centered clipping in G's dtype (double inputs, more than 32 workers on a device), from the [d] `center`, updated in place:
  rows with a non-finite squared distance are skipped, c_i = 1 if sqrt(D_i) <= tau else tau / sqrt(D_i),
  z = z + (sum c_i (x_i - z)) / n with the sum over the kept rows in ascending order and n all the rows; no kept row keeps z."""
  iterations, tau = check_centered_clipping(G.shape[0], 0, iterations, tau)
  n = G.shape[0]
  scalar = lambda value: torch.tensor(value, dtype=G.dtype, device=G.device)
  one, radius, count = scalar(1.0), scalar(tau), scalar(float(n))
  z = center.to(device=G.device, dtype=G.dtype, copy=True)
  dists = []
  for _ in range(iterations):
    delta = G - z.unsqueeze(0)
    D = (delta * delta).sum(dim=1)
    dists.append(D)
    kept = [i for i in range(n) if math.isfinite(float(D[i]))]
    if not kept:
      continue
    # the square root of an fp32 value taken in fp64 and rounded once is correctly rounded (torch's CPU fp32 sqrt is not always)
    root = torch.sqrt(D.double()).to(G.dtype)
    clip = torch.where(root <= radius, one, radius / root)
    u = torch.zeros_like(z)
    for i in kept:
      u = u + clip[i] * (G[i] - z)
    z = z + u / count
  center.copy_(z)
  return (z, torch.stack(dists)) if return_distances else z


def torch_pairwise_distances(G):
  n = G.shape[0]
  dist = torch.zeros((n, n), dtype=G.dtype, device=G.device)
  for i in range(n - 1):
    delta = G[i + 1:] - G[i].unsqueeze(0)
    row = (delta * delta).sum(dim=1)
    row = torch.where(torch.isfinite(row), row, torch.full_like(row, float("inf")))
    dist[i, i + 1:] = row
    dist[i + 1:, i] = row
  return dist


# ---------------------------------------------------------------------------- #
# Nearest-neighbour mixing (NNM; Allouah et al., "Fixing by Mixing", AISTATS 2023): a pre-aggregation run on the rows before the rule

# "arc+nnm": adaptive robust clipping, then NNM on the clipped rows; "bucketing": means of buckets of s rows, which needs the bucket size s
PRE_AGGREGATIONS = ("none", "nnm", "arc", "arc+nnm", "bucketing")


def check_pre_aggregation(name, bucket_size=None):
  """`--pre-aggregation` value -> the `FusedSpec.mix` it selects (None for "none"). "bucketing" is only complete with its bucket size
  `bucket_size` (checked against n by `check_bucketing`)."""
  if name is None or name == "none":
    return None
  if name not in PRE_AGGREGATIONS:
    raise tools.UserException("Unknown pre-aggregation %r (expected one of %s)" % (name, ", ".join(PRE_AGGREGATIONS)))
  if name == "bucketing" and bucket_size is None:
    raise tools.UserException("Bucketing needs a bucket size s >= 1")
  return name


def check_nnm(n, f):
  if not 0 <= 2 * f < n:
    raise tools.UserException("Nearest-neighbour mixing needs 0 <= 2 f < n (got n = %d, f = %d)" % (n, f))


def nnm_select(dist, f):
  """[n, n] distances -> [n, n] bool matrix, row i marking N_i: i itself and the n - f - 1 other rows first under the ordering
  convention (finite ascending, non-finite last, ties -> lower index), whatever the ties at distance 0."""
  n = dist.shape[0]
  check_nnm(n, f)
  key = _rank_key(dist.detach().to("cpu"))
  member = torch.eye(n, dtype=torch.bool)
  for i in range(n):
    others = torch.tensor([j for j in range(n) if j != i], dtype=torch.int64)
    order = torch.argsort(key[i, others], stable=True)
    member[i, others[order[:n - f - 1]]] = True
  return member


def nnm_bits(member):
  """[n, n] bool neighbourhoods (n <= 32) -> [n] int32 bit masks, the layout the sm_90a kernel reports."""
  values = [sum(1 << j for j in range(member.shape[1]) if bool(member[i, j])) for i in range(member.shape[0])]
  return torch.tensor([v - (1 << 32) if v >= 1 << 31 else v for v in values], dtype=torch.int32)


def _nnm_members(masks, n):
  """Neighbourhoods as an [n, n] bool matrix, from that matrix or from [n] int32 bit masks."""
  masks = masks.detach().to("cpu")
  if masks.dim() == 2:
    return masks.bool()
  return torch.tensor([[(int(masks[i]) >> j) & 1 == 1 for j in range(n)] for i in range(n)], dtype=torch.bool)


def torch_nnm_mix(G, masks, f):
  """y_i = (((x_a0 + x_a1) + x_a2) + ...) / (n - f) over the members of N_i in ascending worker order from +0, in G's dtype: one
  `torch.add` per member and one division by a 0-d tensor (a sum over a gathered index may add in another order)."""
  n = G.shape[0]
  check_nnm(n, f)
  member = _nnm_members(masks, n)
  count = torch.tensor(float(n - f), dtype=G.dtype, device=G.device)
  Y = torch.empty_like(G)
  for i in range(n):
    acc = torch.zeros_like(G[i])
    for j in range(n):
      if bool(member[i, j]):
        acc = torch.add(acc, G[j])
    Y[i] = torch.div(acc, count)
  return Y


def torch_nnm(G, f, return_details=False):
  """NNM with the torch back-end: distances, selection, mixing; `return_details` also gives (distances, [n, n] neighbourhoods)."""
  dist = torch_pairwise_distances(G)
  member = nnm_select(dist, f)
  Y = torch_nnm_mix(G, member, f)
  return (Y, dist, member) if return_details else Y


def host_nnm(G, f):
  """NNM with the host library's distances; selection and mixing on CPU tensors. Returns the mixed rows on G's device."""
  Gc = G.detach().to("cpu").contiguous()
  member = nnm_select(host_pairwise_distances(Gc), f)
  return torch_nnm_mix(Gc, member, f).to(G.device)


# Adaptive robust clipping (ARC; Allouah et al., "Boosting Robustness by Clipping Gradients in Distributed Learning"): the k rows of
# largest norm are clipped to the norm of the largest row left alone

def check_arc(n, f):
  if not 0 <= 2 * f < n:
    raise tools.UserException("Adaptive robust clipping needs 0 <= 2 f < n (got n = %d, f = %d)" % (n, f))


def arc_clip_count(n, f):
  """k = floor(2 f (n - f) / n), in integer arithmetic: the number of rows ARC clips."""
  check_arc(n, f)
  return (2 * f * (n - f)) // n


def arc_factors(N, f):
  """[n] squared row norms -> ([n] factors in N's dtype, [n] bool mask of the clipped rows). The rows are ordered by N (finite ascending,
  non-finite last, ties -> lower index); the last k are clipped, C = sqrt(N) of the row at position n - k - 1, and a clipped row's
  factor is 1 if sqrt(N_i) <= C else C / sqrt(N_i) (every square root and the division rounded once); every factor is 1 and no row
  is clipped when k = 0 or C is not finite."""
  N = N.detach().to("cpu")
  n = N.shape[0]
  k = arc_clip_count(n, f)
  one = torch.tensor(1.0, dtype=N.dtype)
  factors = torch.ones(n, dtype=N.dtype)
  clipped = torch.zeros(n, dtype=torch.bool)
  if k == 0:
    return factors, clipped
  order = torch.argsort(_rank_key(N), stable=True)
  # the square root of an fp32 value taken in fp64 and rounded once is correctly rounded
  root = torch.sqrt(N.double()).to(N.dtype)
  C = root[order[n - k - 1]]
  if not math.isfinite(float(C)):
    return factors, clipped
  for i in order[n - k:].tolist():
    clipped[i] = True
    factors[i] = one if bool(root[i] <= C) else torch.div(C, root[i])
  return factors, clipped


def torch_arc_clip(G, factors):
  """y_i = x_i * c_i, one `torch.mul` per row whose factor is not 1 (NaN included); the other rows are copied unchanged."""
  Y = G.clone()
  factors = factors.detach().to("cpu")
  for i in range(G.shape[0]):
    c = factors[i]
    if not bool(c == 1):
      Y[i] = torch.mul(G[i], c.to(device=G.device, dtype=G.dtype))
  return Y


def torch_arc(G, f, return_details=False):
  """ARC with the torch back-end in G's dtype: squared norms, factors, clipping; `return_details` also gives (N, factors, clipped)."""
  N = (G * G).sum(dim=1)
  factors, clipped = arc_factors(N, f)
  Y = torch_arc_clip(G, factors)
  return (Y, N, factors, clipped) if return_details else Y


def torch_pre_aggregate(G, mix, f, host=False, bucket_size=None, seed=0, step=0):
  """The pre-aggregation `mix` (a `FusedSpec.MIXES` value, or "bucketing") of the [n, d] rows G with the torch reference: ARC, then
  NNM; `host`: NNM takes the host library's distances for CPU rows (`host_nnm`). Bucketing (`bucket_size`, `seed`, `step`) returns
  the n' = ceil(n / s) bucket means."""
  if mix is None:
    return G
  if mix not in PRE_AGGREGATIONS:
    raise tools.UserException("Unknown pre-aggregation %r (expected one of %s)" % (mix, ", ".join(PRE_AGGREGATIONS)))
  if mix == "bucketing":
    return torch_bucketing(G, bucket_size, seed, step)
  if mix in ("arc", "arc+nnm"):
    G = torch_arc(G, f)
  if mix in ("nnm", "arc+nnm"):
    G = host_nnm(G, f) if host and G.device.type == "cpu" else torch_nnm(G, f)
  return G


# Bucketing (Karimireddy, He & Jaggi, "Byzantine-Robust Learning on Heterogeneous Datasets via Bucketing", ICLR 2022): the rows are
# shuffled by a keyed permutation, cut into buckets of s rows and replaced by the n' = ceil(n / s) bucket means

BUCKETING_TAG = 0x42554B54   # "BUKT": the third splitmix64 input of the key; >= 8, so it never equals one of DnC's iteration numbers
_MASK64 = (1 << 64) - 1


def _splitmix64_int(z):
  """splitmix64 on a Python integer, mod 2^64 (the same function as `_splitmix64` and the kernels' `splitmix64`)."""
  z = (z + 0x9E3779B97F4A7C15) & _MASK64
  z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _MASK64
  z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _MASK64
  return z ^ (z >> 31)


def check_bucketing(n, s):
  """1 <= s <= n -> n' = ceil(n / s), the number of buckets (the rows the rule sees)."""
  if isinstance(s, bool) or not isinstance(s, int) or not 1 <= s <= n:
    raise tools.UserException("Bucketing needs a bucket size 1 <= s <= n (got n = %d, s = %r)" % (n, s))
  return (n + s - 1) // s


def check_bucketing_key(seed, step):
  if isinstance(seed, bool) or int(seed) != seed or not 0 <= seed <= _MASK64:
    raise tools.UserException("Bucketing needs a seed in [0, 2^64) (got %r)" % (seed,))
  if isinstance(step, bool) or int(step) != step or not 0 <= step < 1 << 63:
    raise tools.UserException("Bucketing needs a step key in [0, 2^63) (got %r)" % (step,))
  return int(seed), int(step)


def bucketing_permutation(n, seed, step):
  """pi of step `step`, a list of the n worker indices: K = splitmix64(splitmix64(splitmix64(seed) ^ step) ^ TAG); from the identity,
  for i = n - 1 down to 1, j = splitmix64(K ^ i) mod (i + 1) and pi[i], pi[j] are swapped (unsigned 64-bit arithmetic)."""
  seed, step = check_bucketing_key(seed, step)
  key = _splitmix64_int(_splitmix64_int(_splitmix64_int(seed) ^ step) ^ BUCKETING_TAG)
  perm = list(range(n))
  for i in range(n - 1, 0, -1):
    j = _splitmix64_int(key ^ i) % (i + 1)
    perm[i], perm[j] = perm[j], perm[i]
  return perm


def bucketing_masks(n, s, perm):
  """The n' member sets as bit masks (Python ints): bucket b holds pi[b s], ..., pi[min((b + 1) s, n) - 1]."""
  count = check_bucketing(n, s)
  return [sum(1 << perm[p] for p in range(b * s, min((b + 1) * s, n))) for b in range(count)]


def bucketing_mean(G, masks):
  """y_b = (((x_a0 + x_a1) + ...) / |M_b| over the members of every mask in ascending worker order from +0, in G's dtype: one
  `torch.add` per member and one division by a 0-d tensor (NNM's mixing arithmetic). `masks`: ints, or the kernel's int32 values."""
  Y = torch.empty((len(masks),) + tuple(G.shape[1:]), dtype=G.dtype, device=G.device)
  for b, mask in enumerate(masks):
    mask = int(mask) + (1 << 32 if int(mask) < 0 else 0)
    members = [j for j in range(G.shape[0]) if (mask >> j) & 1]
    acc = torch.zeros_like(G[0])
    for j in members:
      acc = torch.add(acc, G[j])
    Y[b] = torch.div(acc, torch.tensor(float(len(members)), dtype=G.dtype, device=G.device))
  return Y


def torch_bucketing(G, s, seed, step, return_details=False):
  """Bucketing of the [n, d] rows G with the torch back-end in G's dtype -> [n', d] bucket means; `return_details` also gives
  (pi [n] int32, masks [n'] int32), the layout the sm_90a kernel reports."""
  n = G.shape[0]
  check_bucketing(n, s)
  perm = bucketing_permutation(n, seed, step)
  masks = bucketing_masks(n, s, perm)
  Y = bucketing_mean(G, masks)
  if not return_details:
    return Y
  return Y, torch.tensor(perm, dtype=torch.int32), torch.tensor([v - (1 << 32) if v >= 1 << 31 else v for v in masks], dtype=torch.int32)


def krum_select(dist, f, m):
  """[n, n] distances -> (scores [n], ids of the m best, ascending score / index-stable)."""
  n = dist.shape[0]
  off = dist.clone()
  off.fill_diagonal_(float("inf"))  # a worker is not its own neighbour
  ranked, _ = torch.sort(_rank_key(off), dim=1, stable=True)
  scores = ranked[:, :n - f - 2].sum(dim=1)
  order = torch.argsort(_rank_key(scores), stable=True)
  return scores, order[:m]


def torch_krum(G, f, m, return_selected=False):
  dist = torch_pairwise_distances(G)
  _, selected = krum_select(dist, f, m)
  selected, _ = torch.sort(selected)
  out = G[selected].sum(dim=0) / m
  return (out, selected) if return_selected else out


def torch_bulyan_weights(dist, f, m):
  """Pure-python transcription of the selection loop (small n): returns the [theta, n] weight matrix."""
  n = dist.shape[0]
  theta = n - 2 * f - 2
  inscore = n - f - 2
  D = dist.detach().to("cpu", torch.float64)
  D = torch.where(torch.isfinite(D), D, torch.full_like(D, float("inf")))
  key = lambda value, index: (0 if value != float("inf") and value == value else 1, value if value == value else 0.0, index)
  pruned = D.clone()
  scores = []
  for i in range(n):
    others = sorted((j for j in range(n) if j != i), key=lambda j: key(float(D[i, j]), j))
    scores.append(sum(float(D[i, j]) for j in others[:inscore]))
    for j in others[inscore:]:
      pruned[i, j] = 0.0
  removed = [False] * n
  weights = torch.zeros((theta, n), dtype=dist.dtype)
  for k in range(theta):
    order = sorted(range(n), key=lambda i: (removed[i],) + key(scores[i], i))
    count = m - k
    for i in order[:count]:
      weights[k, i] = 1.0 / count
    best = order[0]
    removed[best] = True
    for i in range(n):
      if not removed[i]:
        scores[i] -= float(pruned[i, best])
  return weights


def torch_bulyan(G, f, m, return_weights=False):
  n = G.shape[0]
  theta = n - 2 * f - 2
  beta = theta - 2 * f
  dist = torch_pairwise_distances(G)
  weights = torch_bulyan_weights(dist, f, m).to(G.device)
  inter = torch.stack([G[weights[k] != 0].sum(dim=0) / int((weights[k] != 0).sum()) for k in range(theta)], dim=0)
  out = torch_averaged_median(inter, beta)
  return (out, weights) if return_weights else out


# ---------------------------------------------------------------------------- #
# Divide-and-conquer (DnC; Shejwalkar & Houmansadr, "Manipulating the Byzantine", NDSS 2021): the sampler, the selection (a float64
# transcription of the sm_90a kernel's, bit for bit), the torch and host back-ends

DNC_MAX_ITERATIONS = 8
DNC_MAX_SUBSAMPLE = 1 << 20
DNC_MAX_DOMAIN = 1 << 48
DNC_JACOBI_SWEEPS = 32
DNC_JACOBI_TOL = 1e-26
_U64 = (1 << 64) - 1


def check_dnc(n, f, iterations, subsample, c, seed):
  """Validate DnC's parameters -> (iterations, subsample, c, seed, r) with r = floor(c f) computed in float64."""
  if not 0 <= 2 * f < n:
    raise tools.UserException("DnC needs 0 <= 2 f < n (got n = %d, f = %d)" % (n, f))
  if isinstance(iterations, bool) or int(iterations) != iterations or not 1 <= iterations <= DNC_MAX_ITERATIONS:
    raise tools.UserException("DnC needs 1 <= iterations <= %d (got %r)" % (DNC_MAX_ITERATIONS, iterations))
  if isinstance(subsample, bool) or int(subsample) != subsample or not 1 <= subsample <= DNC_MAX_SUBSAMPLE:
    raise tools.UserException("DnC needs 1 <= subsample <= 2^20 (got %r)" % (subsample,))
  c = float(c)
  if not (math.isfinite(c) and c >= 0):
    raise tools.UserException("DnC needs a finite filtering fraction c >= 0 (got %r)" % (c,))
  if isinstance(seed, bool) or int(seed) != seed or not 0 <= seed <= _U64:
    raise tools.UserException("DnC needs a seed in [0, 2^64) (got %r)" % (seed,))
  r = math.floor(c * f)
  if n - int(iterations) * r < 1:
    raise tools.UserException("DnC removes r = floor(c f) = %d rows per iteration: n - iterations * r = %d must be >= 1" % (r, n - int(iterations) * r))
  return int(iterations), int(subsample), c, int(seed), int(r)


def check_dnc_step(step):
  """DnC's step key: an integer in [0, 2^63) (the kernels take it as a signed 64-bit value)."""
  if isinstance(step, bool) or int(step) != step or not 0 <= step < 1 << 63:
    raise tools.UserException("DnC needs a step key in [0, 2^63) (got %r)" % (step,))
  return int(step)


def _splitmix64(z):
  z = z + np.uint64(0x9E3779B97F4A7C15)
  z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
  z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
  return z ^ (z >> np.uint64(31))


def dnc_sample(domain, subsample, seed, step, t):
  """The b' = min(subsample, domain) coordinates of [0, domain) that iteration t of step `step` samples: P(0), ..., P(b' - 1), P a
  4-round Feistel permutation on w bits (w the smallest even number >= max(2, bit length of domain - 1)) with round function
  F_r(R) = splitmix64(K ^ (r << 48) ^ R) mod 2^(w/2), K = splitmix64(splitmix64(splitmix64(seed) ^ step) ^ t), cycle-walked into
  [0, domain). -> int64 array."""
  domain, step = int(domain), check_dnc_step(step)
  if not 1 <= domain <= DNC_MAX_DOMAIN:
    raise tools.UserException("DnC samples a domain of 1 to 2^48 coordinates (got %d)" % domain)
  with np.errstate(over="ignore"):
    key = _splitmix64(np.array([seed & _U64], dtype=np.uint64))
    key = _splitmix64(key ^ np.uint64(step))
    key = _splitmix64(key ^ np.uint64(t))
    width = max(2, (domain - 1).bit_length())
    half = np.uint64((width + (width & 1)) // 2)
    mask = np.uint64((1 << int(half)) - 1)

    def feistel(x):
      L, R = x >> half, x & mask
      for r in range(4):
        L, R = R, L ^ (_splitmix64(key ^ np.uint64(r << 48) ^ R) & mask)
      return (L << half) | R

    y = feistel(np.arange(min(int(subsample), domain), dtype=np.uint64))
    out = y >= np.uint64(domain)
    while out.any():
      y[out] = feistel(y[out])
      out = y >= np.uint64(domain)
  return y.astype(np.int64)


def _serial_sum(values):
  """Left-to-right float64 sum from +0 (np.sum adds pairwise)."""
  return float(np.cumsum(np.concatenate([[0.0], values]))[-1])


def _serial_sums(values):
  """Left-to-right float64 sums from +0 of the rows of the [S, k] array `values` -> [S]."""
  return np.cumsum(np.concatenate([np.zeros((values.shape[0], 1)), values], axis=1), axis=1)[:, -1]


def _jacobi(A, V=None):
  """In place on the stack of symmetric [S, m, m] float64 matrices A (m >= 2) and, when given, their [S, m, m] eigenvector matrices V:
  the cyclic Jacobi of `dnc_eigh`, applied to every matrix on its own. A matrix that passes its stop test is frozen (left out of the
  later sweeps), exactly as if it had been run alone."""
  m = A.shape[1]
  mm = m + (m & 1)
  offdiag = ~np.eye(m, dtype=bool)
  diag = np.arange(m)
  player = lambda pos, rnd: 0 if pos == 0 else 1 + (pos - 1 + rnd) % (mm - 1)
  active = np.arange(A.shape[0])
  with np.errstate(over="ignore", divide="ignore", invalid="ignore"):
    for _ in range(DNC_JACOBI_SWEEPS):
      sq = A[active] * A[active]
      active = active[~(_serial_sums(sq[:, offdiag]) <= DNC_JACOBI_TOL * _serial_sums(sq[:, diag, diag]))]
      if active.size == 0:
        break
      X = A[active]
      W = V[active] if V is not None else None
      for rnd in range(mm - 1):
        pairs = [sorted((player(k, rnd), player(mm - 1 - k, rnd))) for k in range(mm // 2)]
        pairs = [(p, q) for p, q in pairs if q < m]
        P = np.array([p for p, _ in pairs])
        Q = np.array([q for _, q in pairs])
        apq = X[:, P, Q]
        tau = (X[:, Q, Q] - X[:, P, P]) / (2.0 * apq)
        t = np.where(tau >= 0, 1.0, -1.0) / (np.abs(tau) + np.sqrt(1.0 + tau * tau))
        c = 1.0 / np.sqrt(1.0 + t * t)
        s = t * c
        zero = apq == 0
        c, s = np.where(zero, 1.0, c)[:, :, None], np.where(zero, 0.0, s)[:, :, None]
        bp, bq = X[:, P, :].copy(), X[:, Q, :].copy()
        X[:, P, :], X[:, Q, :] = c * bp - s * bq, s * bp + c * bq
        c, s = c.transpose(0, 2, 1), s.transpose(0, 2, 1)
        bp, bq = X[:, :, P].copy(), X[:, :, Q].copy()
        X[:, :, P], X[:, :, Q] = c * bp - s * bq, s * bp + c * bq
        if W is not None:
          vp, vq = W[:, :, P].copy(), W[:, :, Q].copy()
          W[:, :, P], W[:, :, Q] = c * vp - s * vq, s * vp + c * vq
        X[:, P, Q] = 0.0
        X[:, Q, P] = 0.0
      A[active] = X
      if V is not None:
        V[active] = W


def dnc_eigh(B):
  """Float64 cyclic Jacobi on the symmetric [m, m] matrix B (m >= 2) -> (eigenvalues, eigenvectors as columns), the sm_90a kernel's
  operations one for one: before each sweep (at most 32) stop when sum_{i != j} B_ij^2 <= 1e-26 sum_i B_ii^2 (both added row-major);
  a sweep is m' - 1 rounds (m' = m rounded up to even) of m' / 2 disjoint pairs (circle method); a round computes every pair's rotation
  from B as it stands (tau = (B_qq - B_pp) / (2 B_pq), t = sign(tau) / (|tau| + sqrt(1 + tau^2)), c = 1 / sqrt(1 + t^2), s = t c; none
  when B_pq = 0), rotates rows p, q, then columns p, q of B and V, then zeroes B_pq and B_qp."""
  A = np.array(B, dtype=np.float64, copy=True)[None]
  V = np.eye(A.shape[1])[None].copy()
  _jacobi(A, V)
  return np.diag(A[0]).copy(), V[0]


def dnc_scores(dist):
  """Scores u_i^2 of the m rows of the finite [m, m] distance matrix `dist`: u the top eigenvector of the classical double centring
  B = -1/2 (D_ij - r_i - r_j + g) (r_i the row means, g the mean of the r_i, both added in ascending index, float64), from `dnc_eigh`;
  a tie in the top eigenvalue goes to the lower column. m <= 1: zeros."""
  D = np.asarray(dist, dtype=np.float64)
  m = D.shape[0]
  if m <= 1:
    return np.zeros(m)
  r = np.cumsum(np.concatenate([np.zeros((m, 1)), D], axis=1), axis=1)[:, -1] / float(m)
  g = _serial_sum(r) / float(m)
  B = -0.5 * (((D - r[:, None]) - r[None, :]) + g)
  lam, V = dnc_eigh(B)
  u = V[:, int(np.argmax(lam))]
  return u * u


def dnc_select(dists, r):
  """[T, n, n] sampled distances -> ([T, n] bool: the rows iteration t keeps, [n] bool: the rows every iteration kept). Iteration t
  drops the rows with the most non-finite distances to the other remaining rows, the highest index first, until every remaining
  distance is finite (they score +inf); the others score `dnc_scores`; it keeps the n - r rows first under the ordering convention."""
  dists = np.asarray(dists.detach().to("cpu") if isinstance(dists, torch.Tensor) else dists, dtype=np.float64)
  T, n = dists.shape[0], dists.shape[1]
  masks = np.zeros((T, n), dtype=bool)
  for t in range(T):
    D = dists[t]
    bad = ~np.isfinite(D)
    remaining = list(range(n))
    while True:
      counts = [int(bad[i, remaining].sum()) for i in remaining]
      most = max(counts)
      if most == 0:
        break
      remaining.pop(max(k for k, value in enumerate(counts) if value == most))
    scores = np.full(n, np.inf)
    scores[remaining] = dnc_scores(D[np.ix_(remaining, remaining)])
    order = sorted(range(n), key=lambda i: (not np.isfinite(scores[i]), scores[i] if np.isfinite(scores[i]) else 0.0, i))
    masks[t, order[:n - r]] = True
  return masks, masks.all(axis=0)


def selection_mean(G, good):
  """Mean of the rows `good` ([n] bool) of G, added in ascending order from +0 and divided once, in G's dtype (Krum's phase D)."""
  acc = torch.zeros_like(G[0])
  for i in range(G.shape[0]):
    if bool(good[i]):
      acc = torch.add(acc, G[i])
  return torch.div(acc, torch.tensor(float(int(np.sum(good))), dtype=G.dtype, device=G.device))


def torch_dnc(G, f, iterations, subsample, c, seed, step, domain=None, return_details=False):
  """DnC with torch ops in G's dtype and on its device (double inputs, more than 32 workers, the test oracle); `domain` defaults to
  G's row length. `return_details` also gives the [T, n, n] sampled distances and the masks of `dnc_select`."""
  n, d = G.shape
  T, b, _, seed, r = check_dnc(n, f, iterations, subsample, c, seed)
  step = check_dnc_step(step)
  domain = d if domain is None else int(domain)
  if domain > d:
    raise tools.UserException("DnC samples [0, %d) from rows of %d coordinates" % (domain, d))
  dists = []
  for t in range(T):
    index = torch.from_numpy(dnc_sample(domain, b, seed, step, t)).to(G.device)
    dists.append(torch_pairwise_distances(G[:, index]))
  dists = torch.stack(dists)
  masks, good = dnc_select(dists, r)
  out = selection_mean(G, good)
  return (out, dists, (masks, good)) if return_details else out


def host_dnc(G, f, iterations, subsample, c, seed, step, domain=None, return_details=False):
  """DnC with the host library: its sampled distances (`agb_cpu_dnc_sample_distances`), the selection of `dnc_select` and its
  selection mean. Returns the output on G's device."""
  Gc = G.detach().to("cpu").contiguous()
  n, d = Gc.shape
  T, b, _, seed, r = check_dnc(n, f, iterations, subsample, c, seed)
  step = check_dnc_step(step)
  domain = d if domain is None else int(domain)
  if not 1 <= domain <= min(d, DNC_MAX_DOMAIN):
    raise tools.UserException("DnC samples [0, %d) from rows of %d coordinates" % (domain, d))
  dists = torch.empty((T, n, n), dtype=Gc.dtype)
  status = _host("dnc_sample_distances", Gc.dtype)(_ptr(Gc), ctypes.c_size_t(n), ctypes.c_size_t(d), ctypes.c_size_t(T), ctypes.c_size_t(b),
                                                   ctypes.c_uint64(seed), ctypes.c_uint64(step), ctypes.c_size_t(domain), _ptr(dists))
  if status != 0:
    raise tools.UserException("Host DnC rejected its arguments (n = %d, d = %d, iterations = %d, subsample = %d)" % (n, d, T, b))
  masks, good = dnc_select(dists, r)
  selected = torch.tensor([i for i in range(n) if good[i]], dtype=torch.int64)
  out = torch.empty(d, dtype=Gc.dtype)
  status = _host("selection_mean", Gc.dtype)(_ptr(Gc), ctypes.c_size_t(n), ctypes.c_size_t(d), _ptr(selected), ctypes.c_size_t(selected.numel()), _ptr(out))
  if status != 0:
    raise tools.UserException("Host selection mean rejected its arguments")
  out = out.to(G.device)
  return (out, dists, (masks, good)) if return_details else out


# ---------------------------------------------------------------------------- #
# Smallest maximum eigenvalue averaging (SMEA; Allouah et al., "Robust Distributed Learning: Tight Error Bounds and Breakdown Point
# under Data Heterogeneity", NeurIPS 2023): the selection (the sm_90a kernel's, bit for bit), the torch and host back-ends

# the selection costs about 3.4 ms per set of 28 rows and warp on an H100 (every warp of the grid searches its share of the sets): the
# bound keeps it below 50 ms; C(32, 4) = 35960 sets took 114 ms
SMEA_MAX_SETS = 1 << 14


def check_smea(n, f):
  if not 0 <= 2 * f < n:
    raise tools.UserException("SMEA needs 0 <= 2 f < n (got n = %d, f = %d)" % (n, f))
  if math.comb(n, f) > SMEA_MAX_SETS:
    raise tools.UserException("SMEA runs one eigenvalue search per subset of removed workers: C(%d, %d) = %d is above the bound 2^14" % (n, f, math.comb(n, f)))


def smea_scores(dist, f, chunk=2048):
  """[n, n] distances -> float64 scores of the C(n, f) kept sets S (|S| = m = n - f), in lexicographic kept-set order
  (`itertools.combinations`): the largest diagonal entry of B_S = -1/2 (D_ij - r_i - r_j + g) over S (`dnc_scores`' double centring)
  after `dnc_eigh`'s Jacobi, i.e. m times the largest eigenvalue of the covariance of S; +inf when a distance between two members of S
  is not finite; 0 for m = 1. Vectorised over the sets (`chunk` at a time); every value has the bits of `dnc_eigh` on that set alone."""
  D = np.asarray(dist.detach().to("cpu") if isinstance(dist, torch.Tensor) else dist, dtype=np.float64)
  n = D.shape[0]
  check_smea(n, f)
  m = n - f
  sets = np.array(list(itertools.combinations(range(n), m)), dtype=np.int64).reshape(-1, m)
  scores = np.zeros(sets.shape[0])
  for lo in range(0, sets.shape[0], chunk):
    part = sets[lo:lo + chunk]
    DS = D[part[:, :, None], part[:, None, :]]
    finite = np.isfinite(DS).all(axis=(1, 2))
    scores[lo:lo + chunk][~finite] = np.inf
    if m < 2 or not finite.any():
      continue
    DS = DS[finite]
    r = _serial_sums(DS.reshape(-1, m)).reshape(-1, m) / float(m)
    g = _serial_sums(r) / float(m)
    B = -0.5 * (((DS - r[:, :, None]) - r[:, None, :]) + g[:, None, None])
    _jacobi(B)
    with np.errstate(invalid="ignore"):
      scores[lo:lo + chunk][finite] = np.max(np.diagonal(B, axis1=1, axis2=2), axis=1)
  return scores


def smea_select(dist, f, return_score=False):
  """[n, n] distances -> ascending ids of the n - f kept workers whose score (`smea_scores`) is smallest, compared as doubles with
  non-finite scores last and -0 == +0; ties -> the lexicographically smallest id list (`argmin` returns the first minimum of the
  lexicographic enumeration). `return_score` also gives the winning score (+0 for a zero, +inf for a non-finite score)."""
  n = dist.shape[0]
  scores = smea_scores(dist, f)
  key = np.where(np.isfinite(scores), scores, np.inf)
  best = int(np.argmin(key))
  ids = torch.tensor(next(itertools.islice(itertools.combinations(range(n), n - f), best, None)), dtype=torch.int64)
  return (ids, float(key[best]) + 0.0) if return_score else ids


def torch_smea(G, f, return_details=False):
  """SMEA with torch ops in G's dtype and on its device (double inputs, more than 32 workers, the test oracle): distances, the selection
  of `smea_select`, the selection mean. `return_details` also gives (distances, selected ids, winning score)."""
  n = G.shape[0]
  check_smea(n, f)
  dist = torch_pairwise_distances(G)
  ids, score = smea_select(dist, f, return_score=True)
  good = np.zeros(n, dtype=bool)
  good[ids.numpy()] = True
  out = selection_mean(G, good)
  return (out, dist, ids, score) if return_details else out


def host_smea(G, f, return_details=False):
  """SMEA with the host library: its distances (`agb_cpu_pairwise_distances`), the selection of `smea_select` and its selection mean.
  Returns the output on G's device; `return_details` also gives (distances, selected ids, winning score)."""
  Gc = G.detach().to("cpu").contiguous()
  n, d = Gc.shape
  check_smea(n, f)
  dist = host_pairwise_distances(Gc)
  ids, score = smea_select(dist, f, return_score=True)
  out = torch.empty(d, dtype=Gc.dtype)
  status = _host("selection_mean", Gc.dtype)(_ptr(Gc), ctypes.c_size_t(n), ctypes.c_size_t(d), _ptr(ids), ctypes.c_size_t(ids.numel()), _ptr(out))
  if status != 0:
    raise tools.UserException("Host selection mean rejected its arguments")
  out = out.to(G.device)
  return (out, dist, ids, score) if return_details else out


# ---------------------------------------------------------------------------- #
# FLTrust (Cao, Fang, Liu & Gong, "FLTrust: Byzantine-robust Federated Learning via Trust Bootstrapping", NDSS 2021): every row is
# weighted by the ReLU of its cosine with a trusted root gradient r and rescaled to r's norm.
#
# The arithmetic every back-end shares:
#   1. fp32 sums P_i = <x_i, r>, N_i = ||x_i||^2, N0 = ||r||^2 (fold order engine-dependent, as every rule's distances);
#   2. from those sums, in float64 with every operation rounded once, in this order:
#        t_i  = P_i / (sqrt(N_i) * sqrt(N0));
#        TS_i = t_i if t_i is finite and > 0, else 0 (also a non-finite row, N_i = 0, N0 = 0, a non-finite root);
#        S    = sum TS_i, added in worker order from +0;
#        a_i  = ((TS_i * sqrt(N0)) / sqrt(N_i)) / S, rounded once to the rows' type (fp32, or float64 for double rows);
#        every a_i = 0 when S = 0;
#   3. y = sum a_i * x_i, from +0 in worker order, every product and sum rounded once (no FMA); rows with a_i = 0 are skipped, so a
#      NaN row contributes nothing and y = +0 when S = 0.
# Given the sums, every back-end produces the same bits. f is not used (any 0 <= f < n). ||y|| <= ||r|| up to rounding: y is a convex
# combination of rows of norm ||r||.

FLTRUST_ROOT_SIZE = 100   # the paper's root dataset size


def check_fltrust(n, f, root_size=FLTRUST_ROOT_SIZE):
  """Validate FLTrust's parameters -> the root dataset size (an integer >= 1). f is not used but must satisfy 0 <= f < n."""
  if not 0 <= f < n:
    raise tools.UserException("FLTrust needs 0 <= f < n (got n = %d, f = %d)" % (n, f))
  if isinstance(root_size, bool) or not isinstance(root_size, int) or root_size < 1:
    raise tools.UserException("FLTrust needs a root dataset of root-size >= 1 samples (got %r)" % (root_size,))
  return root_size


def fltrust_coefficients(P, N, N0, dtype=np.float32):
  """The fp32 sums P [n], N [n] and N0 -> (TS [n] float64, S, a [n] of `dtype`), as stated above (NumPy float64, one rounding per
  operation; np.sqrt is correctly rounded)."""
  P = np.asarray(P, dtype=np.float64).reshape(-1)
  N = np.asarray(N, dtype=np.float64).reshape(-1)
  N0 = np.float64(np.asarray(N0, dtype=np.float64).reshape(-1)[0])
  with np.errstate(all="ignore"):
    s0 = np.sqrt(N0)
    sn = np.sqrt(N)
    t = P / (sn * s0)
    TS = np.where(np.isfinite(t) & (t > 0), t, 0.0)
    S = _serial_sum(TS)
    a = np.zeros(len(P), dtype=dtype)
    if S != 0.0:
      keep = TS > 0
      a[keep] = (((TS[keep] * s0) / sn[keep]) / S).astype(dtype)
  return TS, S, a


def fltrust_weighted_sum(G, a):
  """y = sum a_i * x_i over the rows with a_i != 0, from +0 in worker order, one `torch.mul` and one `torch.add` per row (G's dtype)."""
  out = torch.zeros(G.shape[1], dtype=G.dtype, device=G.device)
  for i, coef in enumerate(np.asarray(a).tolist()):
    if coef != 0.0:
      out = torch.add(out, torch.mul(G[i], torch.tensor(coef, dtype=G.dtype, device=G.device)))
  return out


def check_fltrust_root(G, root):
  """The root gradient of the [n, d] rows G: a [d] tensor, returned in G's dtype on G's device."""
  if root is None:
    raise tools.UserException("FLTrust needs the root gradient r (root=)")
  if root.shape != (G.shape[1],):
    raise tools.UserException("FLTrust needs a [%d] root gradient (got %s)" % (G.shape[1], tuple(root.shape)))
  return root.to(device=G.device, dtype=G.dtype)


def torch_fltrust(G, root, sums=None, return_details=False):
  """FLTrust with the torch back-end in G's dtype. `sums`: (P, N, N0) to use instead of the torch sums (e.g. the kernel's).
  `return_details` also gives (P, N, N0, a)."""
  r = check_fltrust_root(G, root)
  if sums is None:
    P, N, N0 = (G * r).sum(dim=1), (G * G).sum(dim=1), (r * r).sum()
    sums = tuple(v.detach().cpu().numpy() for v in (P, N, N0))
  P, N, N0 = sums
  dtype = np.float64 if G.dtype == torch.float64 else np.float32
  _, _, a = fltrust_coefficients(P, N, N0, dtype)
  out = fltrust_weighted_sum(G, a)
  return (out, P, N, N0, a) if return_details else out


def host_fltrust_sums(G, root):
  """(P [n], N [n], N0) of the [n, d] rows G and the root with the host library (`agb_cpu_fltrust_sums`), as NumPy arrays of G's type."""
  Gc = G.detach().to("cpu").contiguous()
  rc = check_fltrust_root(Gc, root).contiguous()
  n, d = Gc.shape
  out = torch.zeros(2 * n + 1, dtype=Gc.dtype)
  if _host("fltrust_sums", Gc.dtype)(_ptr(Gc), ctypes.c_size_t(n), ctypes.c_size_t(d), _ptr(rc), _ptr(out)) != 0:
    raise tools.UserException("Host FLTrust sums rejected their arguments (n = %d, d = %d)" % (n, d))
  out = out.numpy()
  return out[:n], out[n:2 * n], out[2 * n]


def host_fltrust(G, root, sums=None, return_details=False):
  """FLTrust with the host library: its sums (or `sums`), `fltrust_coefficients`, then `agb_cpu_weighted_sum` (the same skipped rows
  and order as `fltrust_weighted_sum`). Returns the output on G's device; `return_details` also gives (P, N, N0, a)."""
  Gc = G.detach().to("cpu").contiguous()
  n, d = Gc.shape
  P, N, N0 = host_fltrust_sums(Gc, root) if sums is None else sums
  dtype = np.float64 if Gc.dtype == torch.float64 else np.float32
  _, _, a = fltrust_coefficients(P, N, N0, dtype)
  out = _host_weighted_sum(Gc, a).to(G.device)
  return (out, P, N, N0, a) if return_details else out


def _host_weighted_sum(Gc, a):
  """`agb_cpu_weighted_sum` of the contiguous CPU rows Gc with the weights a (Gc's type): the rows and order of `fltrust_weighted_sum`."""
  n, d = Gc.shape
  weights = torch.from_numpy(np.ascontiguousarray(a))
  out = torch.empty(d, dtype=Gc.dtype)
  if _host("weighted_sum", Gc.dtype)(_ptr(Gc), ctypes.c_size_t(n), ctypes.c_size_t(d), _ptr(weights), _ptr(out)) != 0:
    raise tools.UserException("Host weighted sum rejected its arguments")
  return out


# ---------------------------------------------------------------------------- #
# FoolsGold (Fung, Yoon & Beschastnikh, "The Limitations of Federated Learning in Sybil Settings", RAID 2020): every worker i keeps a
# history H_i, the sum of the rows it has submitted; workers whose histories point the same way as another worker's get low weight.
#
# The arithmetic every back-end shares (rows g_i in worker order, histories H_i fp32 from +0):
#   1. H_ik <- H_ik + g_ik (one fp32 add) where g_ik is finite; H_ik is unchanged where it is not, and row i is *bad* this step;
#   2. fp32 sums P_ij = <H_i, H_j> for i <= j of the updated histories, N_i = P_ii (fold order engine-dependent);
#   3. from those sums, in float64 with every operation rounded once (`foolsgold_coefficients`):
#        cs_ij = P_ij / (sqrt(N_i) * sqrt(N_j)) for i != j; 0 when N_i or N_j is 0 or non-finite, or the quotient is non-finite; cs_ii = 0;
#        v_i = max_j cs_ij (>= 0: the diagonal counts);
#        pardoning: cs_ij <- (cs_ij * v_i) / v_j for i != j with v_j > v_i;
#        alpha_i = clip(1 - max_j cs_ij, 0, 1);
#        every c_i = 0 when max alpha = 0; otherwise alpha <- alpha / max alpha, 1 becomes 0.99, alpha <- kappa (ln(alpha / (1 - alpha))
#        + 0.5) (-inf -> 0), clipped to [0, 1];
#        alpha_i = 0 for the bad rows and the rows of non-finite N_i; S = sum alpha_i in worker order from +0;
#        c_i = alpha_i / S rounded once to the rows' type, every c_i = 0 when S = 0;
#   4. y = sum c_i g_i, FLTrust's weighted sum (`fltrust_weighted_sum`): from +0 in worker order, no FMA, the rows of c_i = 0 skipped.
# Given the sums, every back-end produces the same bits (the logarithm is the platform's: CUDA's and the C library's double `log` are
# within 1 ulp of each other, which changes an fp32 c_i only when alpha_i / S lies within that distance of an fp32 rounding boundary).
# f is not used (any 0 <= f < n). kappa is the paper's confidence parameter.

FOOLSGOLD_CONFIDENCE = 1.0   # kappa, as in the authors' code


def check_foolsgold(n, f, confidence=FOOLSGOLD_CONFIDENCE):
  """Validate FoolsGold's parameters -> the confidence kappa (a finite float > 0). f is not used but must satisfy 0 <= f < n."""
  if not 0 <= f < n:
    raise tools.UserException("FoolsGold needs 0 <= f < n (got n = %d, f = %d)" % (n, f))
  try:
    kappa = float(confidence) if not isinstance(confidence, bool) else float("nan")
  except (TypeError, ValueError):
    kappa = float("nan")
  if not (math.isfinite(kappa) and kappa > 0):
    raise tools.UserException("FoolsGold needs a finite confidence > 0 (got %r)" % (confidence,))
  return kappa


def _unit_clip(x):
  """clip(x, 0, 1) with +0 below (x float64 array, no NaN)."""
  return np.where(x > 0.0, np.where(x < 1.0, x, 1.0), 0.0)


def foolsgold_coefficients(P, N, bad, kappa, dtype=np.float32):
  """The fp32 sums P [n, n] (symmetric; N_i = P_ii is taken from N [n]) and the bad-row flags [n] -> (alpha [n] float64, S, c [n] of
  `dtype`), as stated above (NumPy float64, one rounding per operation)."""
  N = np.asarray(N, dtype=np.float64).reshape(-1)
  n = len(N)
  P = np.asarray(P, dtype=np.float64).reshape(n, n)
  bad = np.asarray(bad).reshape(-1).astype(bool)
  kappa = np.float64(kappa)
  with np.errstate(all="ignore"):
    sn = np.sqrt(N)
    ok = np.isfinite(N) & (N != 0.0)
    cs = P / (sn[:, None] * sn[None, :])
    cs = np.where(ok[:, None] & ok[None, :] & np.isfinite(cs), cs, 0.0)
    np.fill_diagonal(cs, 0.0)
    v = cs.max(axis=1)
    cs = np.where(v[None, :] > v[:, None], (cs * v[:, None]) / v[None, :], cs)
    alpha = _unit_clip(1.0 - cs.max(axis=1))
    top = alpha.max()
    c = np.zeros(n, dtype=dtype)
    if top == 0.0:
      return np.zeros(n), 0.0, c
    alpha = alpha / top
    alpha = np.where(alpha == 1.0, 0.99, alpha)
    alpha = _unit_clip(kappa * (np.log(alpha / (1.0 - alpha)) + 0.5))
    alpha = np.where(bad | ~np.isfinite(N), 0.0, alpha)
    S = _serial_sum(alpha)
    if S != 0.0:
      c = (alpha / S).astype(dtype)
  return alpha, S, c


def check_foolsgold_history(G, history):
  """The [n, d] history of the [n, d] rows G: of G's dtype, on G's device (it is updated in place)."""
  if history is None:
    raise tools.UserException("FoolsGold needs the per-worker history H (history=)")
  if tuple(history.shape) != tuple(G.shape) or history.dtype != G.dtype or history.device != G.device:
    raise tools.UserException("FoolsGold needs a %s history of type %s on %s (got %s, %s on %s)" % (
      tuple(G.shape), G.dtype, G.device, tuple(history.shape), history.dtype, history.device))
  return history


def torch_foolsgold(G, history, confidence=FOOLSGOLD_CONFIDENCE, sums=None, return_details=False):
  """FoolsGold with the torch back-end in G's dtype: updates `history` in place, then the sums of the updated histories (or `sums`:
  (P [n, n], N [n], bad [n]), e.g. the kernel's). `return_details` also gives (P, N, bad, c)."""
  H = check_foolsgold_history(G, history)
  finite = torch.isfinite(G)
  H.copy_(torch.where(finite, H + G, H))
  if sums is None:
    P = torch.stack([(H * H[i]).sum(dim=1) for i in range(H.shape[0])]).detach().cpu().numpy()
    sums = P, np.diagonal(P).copy(), (~finite.all(dim=1)).cpu().numpy()
  P, N, bad = sums
  dtype = np.float64 if G.dtype == torch.float64 else np.float32
  _, _, c = foolsgold_coefficients(P, N, bad, confidence, dtype)
  out = fltrust_weighted_sum(G, c)
  return (out, P, N, bad, c) if return_details else out


def host_foolsgold_sums(G, history):
  """The history step and (P [n, n], N [n], bad [n] bool) of the [n, d] rows G with the host library (`agb_cpu_foolsgold_sums`), as
  NumPy arrays of G's type. `history` ([n, d], G's dtype) is updated in place."""
  Gc = G.detach().to("cpu").contiguous()
  n, d = Gc.shape
  H = history if (history.device.type == "cpu" and history.is_contiguous()) else history.detach().to("cpu").contiguous()
  if tuple(H.shape) != (n, d) or H.dtype != Gc.dtype:
    raise tools.UserException("FoolsGold needs a %s history of type %s (got %s, %s)" % ((n, d), Gc.dtype, tuple(H.shape), H.dtype))
  out = torch.zeros(n * n + n, dtype=Gc.dtype)
  if _host("foolsgold_sums", Gc.dtype)(_ptr(Gc), ctypes.c_size_t(n), ctypes.c_size_t(d), _ptr(H), _ptr(out)) != 0:
    raise tools.UserException("Host FoolsGold sums rejected their arguments (n = %d, d = %d)" % (n, d))
  if H is not history:
    history.copy_(H)
  out = out.numpy()
  P = out[:n * n].reshape(n, n)
  return P, np.diagonal(P).copy(), out[n * n:] != 0


def host_foolsgold(G, history, confidence=FOOLSGOLD_CONFIDENCE, sums=None, return_details=False):
  """FoolsGold with the host library: its history step and sums (`sums`, when given, replace the latter), `foolsgold_coefficients`,
  then `agb_cpu_weighted_sum`. Returns the output on G's device; `return_details` also gives (P, N, bad, c)."""
  Gc = G.detach().to("cpu").contiguous()
  own = host_foolsgold_sums(Gc, history)
  P, N, bad = own if sums is None else sums
  dtype = np.float64 if Gc.dtype == torch.float64 else np.float32
  _, _, c = foolsgold_coefficients(P, N, bad, confidence, dtype)
  out = _host_weighted_sum(Gc, c).to(G.device)
  return (out, P, N, bad, c) if return_details else out


# ---------------------------------------------------------------------------- #
# Omniscient Byzantine rows (`attacks/omniscient.py`): the literal definition, the CPU back-end and the oracle of the sm_90a kernel

OPTIMIZED_MODES = ("min-max", "min-sum")   # Shejwalkar & Houmansadr, NDSS 2021: gamma solved from whole-vector sums
DEVIATIONS = ("unit-vec", "sign", "std")
MIMIC_WARMUP = 100   # default number of warm-up steps T0 of mimic
FANG_MODES = ("fang-krum", "fang-trim")   # Fang, Cao, Jia & Gong, USENIX Security 2020: full-knowledge Krum and trimmed-mean attacks
FANG_THRESHOLD = 1e-5   # fang-krum: smallest candidate gamma tested after the first, in gradient units
FANG_SCALE = 2.0   # fang-trim: the paper's b, the width of the interval beyond the extreme honest value
FANG_MAX_CANDIDATES = 64
FANG_TAG = 0x46414E47   # "FANG": the third splitmix64 input of fang-trim's key; >= 8 and != BUCKETING_TAG, so no DnC or bucketing key


def check_byzantine_slots(n, byz_slots, mode):
  """Validated, ascending list of Byzantine slots of an n-row matrix for attack `mode` ("ipm" and "fang-trim" need 1 honest row, the
  others 2)."""
  if mode not in ("alie", "ipm", "mimic") + OPTIMIZED_MODES + FANG_MODES:
    raise tools.UserException("Unknown omniscient attack mode " + repr(mode))
  slots = sorted({int(i) for i in byz_slots})
  if not slots or slots[0] < 0 or slots[-1] >= n:
    raise tools.UserException("Byzantine slots must be a non-empty subset of [0, %d) (got %r)" % (n, list(byz_slots)))
  need = 1 if mode in ("ipm", "fang-trim") else 2
  if n - len(slots) < need:
    raise tools.UserException("%s needs at least %d honest row(s) (n = %d, %d Byzantine)" % (mode.upper(), need, n, len(slots)))
  return slots


def check_deviation(mode, deviation):
  """The deviation of Min-Max / Min-Sum: "unit-vec" (default), "sign" or "std"."""
  if deviation is None:
    return "unit-vec"
  if deviation not in DEVIATIONS:
    raise tools.UserException("%s: unknown deviation %r (expected one of %s)" % (mode, deviation, ", ".join(DEVIATIONS)))
  return deviation


def _scalar(G):
  # divisors are device tensors: a Python-number divisor may be turned into a multiplication by its reciprocal on the GPU
  return lambda value: torch.tensor(value, dtype=torch.float32, device=G.device)


def _honest_mean(honest, scalar):
  """mu = ((h0 + h1) + ...) / H, fp32, one rounded operation at a time."""
  mu = honest[0]
  for h in honest[1:]:
    mu = mu + h
  return mu / scalar(len(honest))


def _honest_sigma(honest, mu, scalar):
  """sqrt(sum_i (h_i - mu)^2 / (H - 1)), same order and rounding as `_honest_mean`."""
  var = None
  for h in honest:
    dev = h - mu
    square = dev * dev
    var = square if var is None else var + square
  # torch's vectorised fp32 sqrt on the CPU is not always correctly rounded: the square root of an fp32 value taken in fp64 and
  # rounded once to fp32 is (fp64 carries more than 2 * 24 + 2 bits)
  return torch.sqrt((var / scalar(len(honest) - 1)).double()).float()


def torch_byzantine_row(G, byz_slots, mode, coef):
  """The row every Byzantine slot receives: per coordinate, from the honest rows h (ascending slots, H of them),
  mu = ((h0 + h1) + ...) / H; ALIE: mu + z * sqrt(sum_i (h_i - mu)^2 / (H - 1)); IPM: (-epsilon) * mu. fp32, one rounded operation at a
  time (separate torch calls, nothing that may fuse into an FMA)."""
  byz = set(check_byzantine_slots(G.shape[0], byz_slots, mode))
  honest = [G[i] for i in range(G.shape[0]) if i not in byz]
  scalar = _scalar(G)
  coef = scalar(coef)
  mu = _honest_mean(honest, scalar)
  if mode == "ipm":
    return torch.neg(coef) * mu
  return mu + coef * _honest_sigma(honest, mu, scalar)


def optimized_deviation(G, byz_slots, mode, deviation):
  """(mu, p) of Min-Max / Min-Sum, fp32 per coordinate: ALIE's mu, and p = mu (unit-vec), sign(mu) (+1, -1, +0 for +-0, NaN for NaN)
  or ALIE's sigma (std)."""
  byz = set(check_byzantine_slots(G.shape[0], byz_slots, mode))
  honest = [G[i] for i in range(G.shape[0]) if i not in byz]
  scalar = _scalar(G)
  mu = _honest_mean(honest, scalar)
  deviation = check_deviation(mode, deviation)
  if deviation == "std":
    return mu, _honest_sigma(honest, mu, scalar)
  if deviation == "sign":
    one = torch.ones_like(mu)
    return mu, torch.where(mu > 0, one, torch.where(mu < 0, -one, torch.where(mu == 0, torch.zeros_like(mu), mu)))
  return mu, mu


def optimized_statistics(G, byz_slots, mode, deviation):
  """(mu, p, A, B, C, T) of Min-Max / Min-Sum: A_i = sum (mu - h_i)^2 and B_i = sum (mu - h_i) p over the honest rows (ascending slots),
  C = sum p^2 and, for Min-Max, T = max_{j<k} sum (h_j - h_k)^2 (None for Min-Sum). The sums are taken in float64 from the fp32 mu, p and
  rows, then rounded once to fp32 (Python floats); a non-finite sum stays non-finite."""
  byz = set(check_byzantine_slots(G.shape[0], byz_slots, mode))
  honest = [G[i] for i in range(G.shape[0]) if i not in byz]
  mu, p = optimized_deviation(G, byz_slots, mode, deviation)
  mu64, p64 = mu.double(), p.double()
  A, B = [], []
  for h in honest:
    dev = mu64 - h.double()
    A.append(fp32(float((dev * dev).sum())))
    B.append(fp32(float((dev * p64).sum())))
  C = fp32(float((p64 * p64).sum()))
  T = None
  if mode == "min-max":
    X = torch.stack(honest).double()
    dist = torch.cat([((X[j + 1:] - X[j]) ** 2).sum(dim=1) for j in range(len(honest) - 1)])
    T = fp32(float(dist.max())) if bool(torch.isfinite(dist).all()) else math.nan
  return mu, p, A, B, C, T


def optimized_gamma(mode, A, B, C, T=None):
  """gamma of Min-Max / Min-Sum from the fp32 sums (Python floats), in float64 with one rounding per operation, rounded once to fp32:
  Min-Max: min_i gamma_i, E_i = max(T - A_i, 0), S_i = sqrt(B_i^2 + C E_i), gamma_i = (B_i + S_i) / C if B_i >= 0 else E_i / (S_i - B_i);
  Min-Sum: sqrt(max_i A_i / C). 0 when C == 0 or any sum is not finite. The sm_90a kernel runs the same operations."""
  values = list(A) + list(B) + [C] + ([T] if mode == "min-max" else [])
  if C == 0 or not all(math.isfinite(v) for v in values):
    return 0.0
  if mode == "min-sum":
    return fp32(math.sqrt(max(A) / C))
  gamma = None
  for a, b in zip(A, B):
    e = max(T - a, 0.0)
    s = math.sqrt(b * b + C * e)
    g = (b + s) / C if b >= 0 else e / (s - b)
    gamma = g if gamma is None else min(gamma, g)
  return fp32(gamma)


def optimized_coefficient(deviation, gamma, C):
  """The push along the deviation's direction: gamma * sqrt(C) for unit-vec (p = mu / ||mu|| in the paper), gamma otherwise."""
  return gamma * math.sqrt(C) if deviation == "unit-vec" and math.isfinite(C) else gamma


def torch_optimized_row(G, byz_slots, mode, deviation, gamma):
  """The Min-Max / Min-Sum row for a given fp32 `gamma`: mu - gamma * p, one rounded fp32 operation at a time (the kernel's arithmetic)."""
  mu, p = optimized_deviation(G, byz_slots, mode, deviation)
  return mu - _scalar(G)(gamma) * p


def torch_craft_byzantine_(G, byz_slots, mode, coef=None, deviation=None, return_details=False, f=None, threshold=None, scale=None, seed=None,
                           step=None):
  """In place on the [n, d] fp32 matrix G: every Byzantine row <- `torch_byzantine_row` (ALIE, IPM) or, for Min-Max / Min-Sum, the row
  of `torch_optimized_row` with the gamma of `optimized_gamma`; honest rows are not written. Min-Max / Min-Sum with `return_details`
  return (gamma, A, B, C, T) instead of G. fang-krum (declared `f`, `threshold`) writes (-gamma) * sign(mu) with the gamma of
  `fang_krum_gamma` and with `return_details` returns (gamma, selected, t, gamma_max, A, B, C, T); fang-trim (`scale`, `seed`, `step`)
  writes every Byzantine row k its own `torch_fang_trim_row`."""
  if G.dtype != torch.float32:
    raise tools.UserException("Omniscient attacks craft fp32 rows (got %s)" % G.dtype)
  if mode == "fang-krum":
    slots = check_byzantine_slots(G.shape[0], byz_slots, mode)
    threshold = check_fang_krum(G.shape[0], len(slots), f, threshold)
    mu, p, A, B, C, T = fang_krum_statistics(G, slots)
    gamma, selected, t, gamma_max = fang_krum_gamma(A, B, C, T, G.shape[0], f, slots, threshold)
    row = torch.neg(_scalar(G)(gamma)) * p
    for i in slots:
      G[i].copy_(row)
    return (gamma, selected, t, gamma_max, A, B, C, T) if return_details else G
  if mode == "fang-trim":
    if return_details:
      raise tools.UserException("return_details is for Min-Max / Min-Sum / fang-krum only")
    slots = check_byzantine_slots(G.shape[0], byz_slots, mode)
    key = fang_trim_key(0 if seed is None else seed, step)
    mu, lo, hi = fang_trim_interval(G, slots, check_fang_scale(scale))
    rows = [fang_trim_value(mu, lo, hi, fang_trim_uniform(G.shape[1], k, key, G.device)) for k in slots]
    for k, row in zip(slots, rows):
      G[k].copy_(row)
    return G
  details = None
  if mode in OPTIMIZED_MODES:
    mu, p, A, B, C, T = optimized_statistics(G, byz_slots, mode, deviation)
    gamma = optimized_gamma(mode, A, B, C, T)
    row = mu - _scalar(G)(gamma) * p
    details = (gamma, A, B, C, T)
  elif return_details:
    raise tools.UserException("return_details is for Min-Max / Min-Sum only")
  else:
    row = torch_byzantine_row(G, byz_slots, mode, coef)
  for i in check_byzantine_slots(G.shape[0], byz_slots, mode):
    G[i].copy_(row)
  return details if return_details else G


# Fang, Cao, Jia & Gong ("Local Model Poisoning Attacks to Byzantine-Robust Federated Learning", USENIX Security 2020), full knowledge,
# written on gradient rows: the paper's crafted local model w' = w - lr g' becomes the gradient g'; its lambda becomes gamma = lambda / lr

def check_fang_krum(n, K, f, threshold):
  """-> the fp32 threshold of fang-krum for n rows, K of them Byzantine, the rule's declared f: n - f - 2 >= 1 (Krum's score has a
  term), n - 2K - 1 >= 1 (the paper's bound on lambda), H = n - K >= 2, a finite threshold > 0 (default `FANG_THRESHOLD`)."""
  if isinstance(f, bool) or not isinstance(f, int) or f < 0:
    raise tools.UserException("fang-krum needs the declared number of Byzantine workers f, an integer >= 0 (got %r)" % (f,))
  if n - f - 2 < 1 or n - 2 * K - 1 < 1 or n - K < 2:
    raise tools.UserException("fang-krum needs n - f - 2 >= 1, n - 2 K - 1 >= 1 and at least 2 honest rows (got n = %d, f = %d, K = %d)" % (n, f, K))
  value = fp32(FANG_THRESHOLD if threshold is None else threshold)
  if not math.isfinite(value) or value <= 0:
    raise tools.UserException("fang-krum: the threshold must be finite and > 0 in fp32 (got %r)" % (threshold,))
  return value


def check_fang_scale(scale):
  """-> the fp32 scale beta of fang-trim (default `FANG_SCALE`): finite and > 1."""
  value = fp32(FANG_SCALE if scale is None else scale)
  if not math.isfinite(value) or value <= 1:
    raise tools.UserException("fang-trim: the scale must be finite and > 1 in fp32 (got %r)" % (scale,))
  return value


def _sign(mu):
  """+1, -1, +0 for +-0, NaN for NaN (Min-Max's `sign` deviation)."""
  one = torch.ones_like(mu)
  return torch.where(mu > 0, one, torch.where(mu < 0, -one, torch.where(mu == 0, torch.zeros_like(mu), mu)))


def fang_krum_statistics(G, byz_slots):
  """(mu, p, A, B, C, T) of fang-krum: ALIE's fp32 mu and p = sign(mu) per coordinate; A_i = sum h_i^2 and B_i = sum h_i p over the honest
  rows (ascending slots), C = sum p^2, and T the honest pair distances sum (h_j - h_k)^2, pairs (j, k), j < k, in lexicographic order
  (the kernel's layout). Every sum is taken in float64 from the fp32 values and rounded once to fp32 (Python floats)."""
  byz = set(check_byzantine_slots(G.shape[0], byz_slots, "fang-krum"))
  honest = [G[i] for i in range(G.shape[0]) if i not in byz]
  mu = _honest_mean(honest, _scalar(G))
  p = _sign(mu)
  p64 = p.double()
  X = torch.stack(honest).double()
  A = [fp32(float((h * h).sum())) for h in X]
  B = [fp32(float((h * p64).sum())) for h in X]
  C = fp32(float((p64 * p64).sum()))
  T = [fp32(float(((X[j] - X[k]) ** 2).sum())) for j in range(len(honest)) for k in range(j + 1, len(honest))]
  return mu, p, A, B, C, T


def _ascending_sum(values, count):
  """0 + v_0 + v_1 + ... over the `count` smallest of `values`, ascending, in float64 (one rounding per addition)."""
  total = 0.0
  for v in sorted(values)[:count]:
    total += v
  return total


def fang_krum_gamma(A, B, C, T, n, f, slots, threshold):
  """-> (gamma, selected, t, gamma_max) of fang-krum from the fp32 sums of `fang_krum_statistics` (Python floats; T in pair order), for
  n rows whose Byzantine slots are `slots`, Krum's declared f and the fp32 `threshold`. float64, one rounding per operation (the sm_90a
  kernel runs the same operations):
    gamma_max = min_i R_i / ((n - 2K - 1) sqrt(C)) + max_i sqrt(A_i) / sqrt(C), R_i the ascending sum of the H - 2 smallest sqrt(T_il),
    l != i honest (the paper's bound on lambda, sqrt(C) in place of sqrt(d));
    candidates gamma_t = gamma_max 2^-t, t = 0, 1, ... while t == 0 or gamma_t >= threshold, at most 64; the first one for which Krum
    with f ranks a Byzantine slot first (ascending score, ties to the lower slot) is kept, else the last one tested. Krum sees the n
    rows with distances 0 between Byzantine rows, max(0, (A_i + (2 gamma) B_i) + (gamma gamma) C) between a Byzantine row and honest
    row i, T between honest rows; a score is the ascending sum of the row's n - f - 2 smallest distances.
  gamma is rounded once to fp32. When C == 0 or any sum is not finite: (0.0, False, -1, 0.0), no candidate tested."""
  slots = sorted(int(i) for i in slots)
  K, H = len(slots), n - len(slots)
  threshold = check_fang_krum(n, K, f, threshold)
  values = list(A) + list(B) + [C] + list(T)
  if len(A) != H or len(B) != H or len(T) != H * (H - 1) // 2:
    raise tools.UserException("fang-krum: expected %d A_i, %d B_i and %d pair distances (got %d, %d, %d)" % (H, H, H * (H - 1) // 2, len(A), len(B), len(T)))
  if C == 0 or not all(math.isfinite(v) for v in values):
    return 0.0, False, -1, 0.0
  pair = {}
  at = 0
  for j in range(H):
    for k in range(j + 1, H):
      pair[j, k] = pair[k, j] = float(T[at])
      at += 1
  others = [[pair[i, l] for l in range(H) if l != i] for i in range(H)]
  R = [_ascending_sum([math.sqrt(v) for v in row], H - 2) for row in others]
  root = math.sqrt(C)
  gamma_max = min(R) / (float(n - 2 * K - 1) * root) + max(math.sqrt(a) for a in A) / root
  honest_slots = [i for i in range(n) if i not in set(slots)]
  m = n - f - 2
  tested = None
  for t in range(FANG_MAX_CANDIDATES):
    gamma = gamma_max * 2.0 ** -t
    if t > 0 and not gamma >= threshold:
      break
    tested = (gamma, t)
    D = [(A[i] + (2.0 * gamma) * B[i]) + (gamma * gamma) * C for i in range(H)]
    D = [v if v > 0.0 else 0.0 for v in D]
    best = (_ascending_sum([0.0] * (K - 1) + D, m), slots[0])
    for i, slot in enumerate(honest_slots):
      best = min(best, (_ascending_sum(others[i] + [D[i]] * K, m), slot))
    if best[1] in slots:
      return fp32(gamma), True, t, gamma_max
  return fp32(tested[0]), False, tested[1], gamma_max


def fang_trim_key(seed, step):
  """fang-trim's key K = splitmix64(splitmix64(splitmix64(seed) ^ step) ^ FANG_TAG): seed in [0, 2^64), step (the number of the update
  the rows feed) in [0, 2^63)."""
  if not isinstance(seed, (int, np.integer)) or isinstance(seed, bool) or not 0 <= seed <= _MASK64:
    raise tools.UserException("fang-trim needs a seed in [0, 2^64) (got %r)" % (seed,))
  if not isinstance(step, (int, np.integer)) or isinstance(step, bool) or not 0 <= step < 1 << 63:
    raise tools.UserException("fang-trim needs a step key in [0, 2^63) (got %r)" % (step,))
  return _splitmix64_int(_splitmix64_int(_splitmix64_int(int(seed)) ^ int(step)) ^ FANG_TAG)


def fang_trim_uniform(d, slot, key, device="cpu"):
  """u of Byzantine slot `slot` at the coordinates [0, d): (splitmix64(K ^ (x 32 + slot)) >> 40) 2^-24, an fp32 [d] tensor (exact)."""
  with np.errstate(over="ignore"):
    index = np.arange(d, dtype=np.uint64) * np.uint64(32) + np.uint64(slot)
    z = _splitmix64(np.uint64(key) ^ index)
  return torch.from_numpy((z >> np.uint64(40)).astype(np.float32) * np.float32(2.0 ** -24)).to(device)


def fang_trim_interval(G, byz_slots, scale):
  """(mu, lo, hi) of fang-trim per coordinate, fp32, one rounded operation at a time: ALIE's mu over the honest rows h (ascending slots);
  mu > 0: e = min_i h_i, [lo, hi] = [e beta, e] if e <= 0 else [e / beta, e]; mu < 0: e = max_i h_i, [lo, hi] = [e, e beta] if e >= 0
  else [e, e / beta]. The minimum and maximum are taken in ascending slot order, a later value replacing the running one only when
  strictly smaller (larger). lo and hi are meaningless where mu is +-0 or NaN."""
  byz = set(check_byzantine_slots(G.shape[0], byz_slots, "fang-trim"))
  honest = [G[i] for i in range(G.shape[0]) if i not in byz]
  scalar = _scalar(G)
  mu = _honest_mean(honest, scalar)
  low, high = honest[0], honest[0]
  for h in honest[1:]:
    low = torch.where(h < low, h, low)
    high = torch.where(h > high, h, high)
  beta = scalar(scale)
  pos = mu > 0
  e = torch.where(pos, low, high)
  scaled, shrunk = e * beta, e / beta
  lo = torch.where(pos, torch.where(e <= 0, scaled, shrunk), e)
  hi = torch.where(pos, e, torch.where(e >= 0, scaled, shrunk))
  return mu, lo, hi


def fang_trim_value(mu, lo, hi, u):
  """b = lo + u (hi - lo), fp32 with one rounding per operation; b = mu where mu is +-0 or NaN."""
  b = lo + u * (hi - lo)
  return torch.where((mu > 0) | (mu < 0), b, mu)


def torch_fang_trim_row(G, byz_slots, slot, scale, key):
  """The fang-trim row of Byzantine slot `slot` of the [n, d] fp32 matrix G, with scale beta and key K (`fang_trim_key`): per coordinate
  x, b = lo + u (hi - lo) over `fang_trim_interval`, u = `fang_trim_uniform`; b = mu where mu is +-0 or NaN. The row is pushed past
  every honest value, against the sign of the mean."""
  mu, lo, hi = fang_trim_interval(G, byz_slots, check_fang_scale(scale))
  return fang_trim_value(mu, lo, hi, fang_trim_uniform(G.shape[1], slot, key, G.device))


def check_mimic(n, byz_slots, warmup):
  """-> (ascending Byzantine slots, T0) of mimic: at least 2 honest rows, an integer warm-up T0 >= 1 (below 2^24, so that the kernel's fp32
  t is exact)."""
  slots = check_byzantine_slots(n, byz_slots, "mimic")
  if isinstance(warmup, bool) or not isinstance(warmup, int) or not 1 <= warmup < 1 << 24:
    raise tools.UserException("mimic: the warm-up must be an integer in [1, 2^24) (got %r)" % (warmup,))
  return slots, warmup


def mimic_state(d, device="cpu", mask=None, real=None):
  """The state of mimic before its first step over [d] rows whose real coordinates are `mask` (a [d] bool tensor; None: all of them):
  t = 0, z = the fp32 of 1 / sqrt(real) on the real coordinates and 0 on the others, i* = -1 (no target yet: the first honest slot).
  `real` defaults to the number of real coordinates; a state that holds only some of the coordinates passes the total."""
  if real is None:
    real = d if mask is None else int(mask.sum())
  if real < 1:
    raise tools.UserException("mimic needs at least one real coordinate")
  z = torch.zeros(d, dtype=torch.float32, device=device)
  value = fp32(1.0 / math.sqrt(real))
  if mask is None:
    z.fill_(value)
  else:
    z[mask.to(device)] = value
  return {"t": 0, "z": z, "istar": torch.full((1,), -1, dtype=torch.int32, device=device)}


def mimic_target(istar, honest):
  """The slot i* designates among the ascending `honest` slots: itself when it is one, the first honest slot otherwise."""
  return istar if istar in honest else honest[0]


def torch_mimic_step_(G, byz_slots, state, warmup, return_details=False):
  """Mimic (Karimireddy, He & Jaggi, ICLR 2022) on the [n, d] fp32 matrix G, in place: every Byzantine row <- the honest row h_{i*}.
  While state["t"] < warmup, one update of the online power iteration first, on the honest rows h (ascending slots, H of them):
  mu = `_honest_mean`, s_i = sum_j (h_i - mu)_j z_j, u = (s_0 (h_0 - mu) + s_1 (h_1 - mu) + ...) / H, y = (t z + u) / (t + 1) (fp32, one
  rounded operation at a time), then, unless ||y||^2 is 0 or not finite, z <- y * (1 / ||y||) and i* <- argmax_i q_i, q_i = sum_j h_i,j y_j
  (ties: lower slot; non-finite q never wins; none finite: the first honest slot); t <- t + 1 in every case. The whole-vector sums are
  float64 sums of the fp32 values; s_i and 1 / ||y|| are rounded once to fp32. `state` (`mimic_state`) is updated in place. With
  `return_details`, returns (s, q, ||y||^2, 1 / ||y||) of the warm-up update (None after the warm-up) instead of G."""
  if G.dtype != torch.float32:
    raise tools.UserException("Omniscient attacks craft fp32 rows (got %s)" % G.dtype)
  n = G.shape[0]
  slots, warmup = check_mimic(n, byz_slots, warmup)
  honest_ids = [i for i in range(n) if i not in set(slots)]
  details = None
  t = int(state["t"])
  if t < warmup:
    honest = [G[i] for i in honest_ids]
    scalar = _scalar(G)
    mu = _honest_mean(honest, scalar)
    devs = [h - mu for h in honest]
    z = state["z"]
    z64 = z.double()
    s = [fp32(float((dev.double() * z64).sum())) for dev in devs]
    acc = None
    for si, dev in zip(s, devs):
      term = scalar(si) * dev
      acc = term if acc is None else acc + term
    y = (scalar(float(t)) * z + acc / scalar(len(honest))) / scalar(float(t + 1))
    y64 = y.double()
    norm2 = float((y64 * y64).sum())
    q = [float((h.double() * y64).sum()) for h in honest]
    inv = 0.0
    if norm2 > 0 and math.isfinite(norm2):
      inv = fp32(1.0 / math.sqrt(norm2))
      z.copy_(y * scalar(inv))
      best = None
      for k, value in enumerate(q):
        if math.isfinite(value) and (best is None or value > q[best]):
          best = k
      state["istar"].fill_(honest_ids[0 if best is None else best])
    state["t"] = t + 1
    details = (s, q, norm2, inv)
  target = mimic_target(int(state["istar"][0]), honest_ids)
  for i in slots:
    G[i].copy_(G[target])
  return details if return_details else G


# ---------------------------------------------------------------------------- #
# Worker momentum (El Mhamdi et al., "Distributed Momentum for Byzantine-resilient SGD"): the CPU back-end and the oracle of the kernel

def torch_worker_momentum_(G, M, beta, c):
  """In place on the [w, d] rows G and momenta M: M <- beta * M + c * G, then G <- M, in G's dtype with one rounding per operation:
  separate `torch.mul` / `torch.add` calls on 0-d tensors of the coefficients (CPU `add_(alpha=)` and `addcmul` may contract to FMA)."""
  if G.shape != M.shape or G.dtype != M.dtype:
    raise tools.UserException("Worker momentum needs rows and momenta of the same shape and type (got %s %s, %s %s)" % (
      tuple(G.shape), G.dtype, tuple(M.shape), M.dtype))
  scalar = lambda value: torch.tensor(value, dtype=G.dtype, device=G.device)
  M.copy_(torch.add(torch.mul(M, scalar(beta)), torch.mul(G, scalar(c))))
  G.copy_(M)
  return G


# ---------------------------------------------------------------------------- #
# Stand-alone CUDA back-end (native/op_gar)

def cuda_aggregate(spec, G):
  """Run the stand-alone sm_90a kernel for `spec` on the [n, d] CUDA matrix G."""
  from ..ops import gar as gar_ops
  return gar_ops.aggregate(spec, G)


def dispatch(G, host_fn, cuda_spec):
  """Default placement policy: CUDA tensors -> sm_90a kernel, CPU tensors -> host C++ library."""
  if G.is_cuda:
    return cuda_aggregate(cuda_spec, G)
  return host_fn(G)
