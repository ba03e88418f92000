"""float64 references of the segmentation U-Net's focal and Dice losses (UNetTrainer(loss=...),
csrc/elementwise.cu seg_dice_stats / seg_loss_grad), in closed form, used by
tests/test_gpu_seg_losses.py and checked against torch.autograd by tests/test_seg_losses_host.py.

Every function takes float64 logits ``l`` [P, >= V] (channels >= V are ignored), int labels ``y``
[P], the class count V, ``w`` None or float64 class weights [V] and ``ignore`` None or the ignored
label value.  S is the set of pixels whose label is not ``ignore``; a label outside [0, V) that is
not ignored is in S with weight 1.
"""
import torch


def pixel_scale(y, V, w=None, ignore=None, options=None):
  """s_p, the cross-entropy's per-pixel factor: 1 / P without loss options, otherwise
  w[y] / sum_S w[y] on S (0 off S, and everywhere when that sum is 0).  ``options`` (default:
  either of w, ignore given) selects the optioned normalisation."""
  P = len(y)
  if options is None:
    options = w is not None or ignore is not None
  if not options:
    return torch.full((P,), 1.0 / P, dtype=torch.float64)
  ok = (y >= 0) & (y < V)
  wy = torch.ones(P, dtype=torch.float64)
  if w is not None:
    wy = torch.where(ok, w.double()[y.clamp(0, V - 1).long()], wy)
  if ignore is not None:
    wy[y == ignore] = 0.0
  sw = float(wy.sum())
  return wy / sw if sw > 0 else torch.zeros(P, dtype=torch.float64)


def _softmax_parts(l, y, V):
  """p [P, V], in-range mask, one-hot [P, V], p_y, q = sum_{j != y} p_j (not 1 - p_y) and
  log p_y accurate also where q is tiny."""
  v = l[:, :V].double()
  ok = (y >= 0) & (y < V)
  yc = y.clamp(0, V - 1).long()
  e = torch.exp(v - v.max(dim=1, keepdim=True).values)
  se = e.sum(dim=1)
  onehot = torch.zeros_like(v)
  onehot[ok, yc[ok]] = 1.0
  ey = (e * onehot).sum(dim=1)
  q = (e * (1.0 - onehot)).sum(dim=1) / se
  py = ey / se
  lp = torch.where(q < 0.5, torch.log1p(-q), v.gather(1, yc[:, None])[:, 0] - torch.logsumexp(v, 1))
  return e / se[:, None], ok, onehot, py, q, lp


def focal_factor(py, q, lp, gamma):
  """(F, q^gamma): the focal gradient factor q^gamma (1 - gamma p_y log(p_y) / q) with its limits
  (q = 0: 1 at gamma = 0, else 0; p_y = 0: q^gamma), and the loss factor q^gamma (0^0 = 1)."""
  qg = torch.where(q > 0, q.clamp_min(1e-300) ** gamma,
                   torch.full_like(q, 1.0 if gamma == 0 else 0.0))
  r = torch.where(q > 0, -lp / q.clamp_min(1e-300), torch.ones_like(q))
  return qg * (1.0 + gamma * py * r), qg


def focal(l, y, V, gamma, w=None, ignore=None, options=None):
  """(loss, dlogits [P, V]) of the focal loss: sum_p s_p q^gamma (-log p_y) and
  s_p (p - onehot) F.  A label outside [0, V) has F = 1 and the cross-entropy term
  logsumexp - 0 (the 8-channel kernel's reading of a padding channel is not modelled)."""
  p, ok, onehot, py, q, lp = _softmax_parts(l, y, V)
  s = pixel_scale(y, V, w, ignore, options)
  F, qg = focal_factor(py, q, lp, gamma)
  F = torch.where(ok, F, torch.ones_like(F))
  qg = torch.where(ok, qg, torch.ones_like(qg))
  term = torch.where(ok, -lp, torch.logsumexp(l[:, :V].double(), 1))
  loss = float((s * qg * term).sum())
  return loss, (s * F)[:, None] * (p - onehot)


def dice_stats(l, y, V, w=None, ignore=None):
  """(I, P, Y) [V] over S."""
  p, ok, onehot, _, _, _ = _softmax_parts(l, y, V)
  S = torch.ones(len(y), dtype=torch.bool) if ignore is None else y != ignore
  return (p * onehot)[S].sum(0), p[S].sum(0), onehot[S].sum(0)


def dice(l, y, V, smooth, w=None, ignore=None):
  """(loss, dlogits [P, V], A [V], B [V]) of the soft multi-class Dice loss over S:
  sum_c omega_c (1 - D_c), D_c = (2 I_c + s) / (P_c + Y_c + s), omega = w / sum w, and its
  gradient p_k (g_k - sum_j p_j g_j) with g_c = A_c [y = c] + B_c, zero off S."""
  p, ok, onehot, _, _, _ = _softmax_parts(l, y, V)
  S = torch.ones(len(y), dtype=torch.bool) if ignore is None else y != ignore
  I, Ps, Y = (p * onehot)[S].sum(0), p[S].sum(0), onehot[S].sum(0)
  wt = torch.ones(V, dtype=torch.float64) if w is None else w.double()
  omega = wt / wt.sum()
  den = Ps + Y + smooth
  D = (2 * I + smooth) / den
  A, B = -2 * omega / den, omega * D / den
  g = onehot * A + B
  d = p * (g - (p * g).sum(1, keepdim=True))
  d[~S] = 0.0
  return float((omega * (1 - D)).sum()), d, A, B
