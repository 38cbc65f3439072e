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
# Omniscient Byzantine rows (`attacks/omniscient.py`): the literal definition, the CPU back-end and the oracle of the sm_90a kernel

def check_byzantine_slots(n, byz_slots, mode):
  """Validated, ascending list of Byzantine slots of an n-row matrix for attack `mode` ("alie" needs 2 honest rows, "ipm" one)."""
  if mode not in ("alie", "ipm"):
    raise tools.UserException("Unknown omniscient attack mode " + repr(mode))
  slots = sorted({int(i) for i in byz_slots})
  if not slots or slots[0] < 0 or slots[-1] >= n:
    raise tools.UserException("Byzantine slots must be a non-empty subset of [0, %d) (got %r)" % (n, list(byz_slots)))
  need = 2 if mode == "alie" else 1
  if n - len(slots) < need:
    raise tools.UserException("%s needs at least %d honest row(s) (n = %d, %d Byzantine)" % (mode.upper(), need, n, len(slots)))
  return slots


def torch_byzantine_row(G, byz_slots, mode, coef):
  """The row every Byzantine slot receives: per coordinate, from the honest rows h (ascending slots, H of them),
  mu = ((h0 + h1) + ...) / H; ALIE: mu + z * sqrt(sum_i (h_i - mu)^2 / (H - 1)); IPM: (-epsilon) * mu. fp32, one rounded operation at a
  time (separate torch calls, nothing that may fuse into an FMA)."""
  byz = set(check_byzantine_slots(G.shape[0], byz_slots, mode))
  honest = [G[i] for i in range(G.shape[0]) if i not in byz]
  # divisors are device tensors: a Python-number divisor may be turned into a multiplication by its reciprocal on the GPU
  scalar = lambda value: torch.tensor(value, dtype=torch.float32, device=G.device)
  coef = scalar(coef)
  mu = honest[0]
  for h in honest[1:]:
    mu = mu + h
  mu = mu / scalar(len(honest))
  if mode == "ipm":
    return torch.neg(coef) * mu
  var = None
  for h in honest:
    dev = h - mu
    square = dev * dev
    var = square if var is None else var + square
  # torch's vectorised fp32 sqrt on the CPU is not always correctly rounded: the square root of an fp32 value taken in fp64 and
  # rounded once to fp32 is (fp64 carries more than 2 * 24 + 2 bits)
  sigma = torch.sqrt((var / scalar(len(honest) - 1)).double()).float()
  return mu + coef * sigma


def torch_craft_byzantine_(G, byz_slots, mode, coef):
  """In place on the [n, d] fp32 matrix G: every Byzantine row <- `torch_byzantine_row`; honest rows are not written."""
  if G.dtype != torch.float32:
    raise tools.UserException("Omniscient attacks craft fp32 rows (got %s)" % G.dtype)
  row = torch_byzantine_row(G, byz_slots, mode, coef)
  for i in check_byzantine_slots(G.shape[0], byz_slots, mode):
    G[i].copy_(row)
  return G


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
