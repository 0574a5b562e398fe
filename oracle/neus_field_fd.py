"""Hand-derived forward/backward of the NeuS SDF field with FINITE-DIFFERENCE normals and Laplacian (VolumeSDF.forward with
grad_type='finite_difference', models/geometry.py:181-199; the Neuralangelo config) in fp64, without autograd -- the CPU restatement of
csrc/neus_field_fd.cu.  The field itself (hash grid with include_xyz + VanillaMLP 35 -> 64 Softplus(100) -> n_out) is that of
oracle/neus_field.py, whose per-level cell / weight rule it reuses.  tests/test_neus_fd_oracle.py checks it against autograd and against
oracle.neus_field.forward at the seven stencil points; tests/helpers/neus_field_fd_ref.py restates it with per-entry error bounds
for the kernel tests (tests/test_gpu_neus_field_fd.py)."""
import torch

from .neus_field import _level_terms
# Stencil point k of a sample: 0 = centre, 1..6 = +x, -x, +y, -y, +z, -z.  Everything is a linear combination of the seven SDF values,
# so the backward is seven ordinary first-order MLP + hash backwards with the upstream gradients
#   centre:  g_out + (g_sdf - 6 g_lap / eps2) e_0;      neighbour a+-:  (+-0.5 g_grad_a / eps + g_lap / eps2) e_0
# Hash levels l >= n_active contribute 0 (ProgressiveBandHashGrid mask) and receive no gradient.

def fd_queries(points, radius, eps):
    """the fp32 unit-cube queries [N,7,3] in the torch path's operation order (models/fields.py): (p + offs).clamp(-r, r) for the
    neighbours, then (q - (-r)) / (r - (-r)) with a true division; the centre is not clamped."""
    p = points.float()
    offs = torch.zeros(6, 3, dtype=torch.float32)
    for a in range(3):
        offs[2 * a, a], offs[2 * a + 1, a] = eps, -eps
    nb = (p[:, None, :] + offs).clamp(-radius, radius)
    q = torch.cat([p[:, None, :], nb], 1)
    return (q - (-radius)) / (radius - (-radius))


def _f32(v):
    """v as the fp32 value the kernels read from fd_state"""
    return float(torch.tensor(float(v), dtype=torch.float32))


def _fd_eval(x01, table, lt, W1, b1, W2, b2, n_active, beta, kernel_cells=False):
    tab = table.double().view(-1, 2)
    feats = []
    for l in range(lt['n_levels']):
        if l < n_active:
            idx, w, _ = _level_terms(x01, tab, lt, l, kernel_cells)
            feats.append((w[..., None] * tab[idx]).sum(1))
        else:
            feats.append(torch.zeros(x01.shape[0], 2, dtype=torch.float64))
    e = torch.cat([x01.double() * 2 - 1] + feats, -1)
    z = e @ W1.double().t() + b1.double()
    h = torch.nn.functional.softplus(z, beta=beta)
    return e, z, h, h @ W2.double().t() + b2.double()


def forward_fd(queries, table, lt, W1, b1, W2, b2, eps, eps2, n_active, beta=100.0, kernel_cells=False):
    """queries [N,7,3] fp32 (fd_queries); eps the step, eps2 the fp32 rounding of eps ** 2 (what torch divides by).
    kernel_cells: every level's cell fraction is the kernels' fp32 pos - floor(pos) (the default takes it from the fp64
    x01 * scale + 0.5), and eps / eps2 are the fp32 values the kernels read from fd_state, so that each of the seven queries of a
    sample interpolates in the kernels' own cell on every level; the rest stays fp64.
    -> sdf [N], grad [N,3], feature [N,n_out], laplace [N], cache."""
    if kernel_cells:
        eps, eps2 = _f32(eps), _f32(eps2)
    N = queries.shape[0]
    x01 = queries.reshape(-1, 3)
    e, z, h, out = _fd_eval(x01, table, lt, W1, b1, W2, b2, n_active, beta, kernel_cells)
    s = out[:, 0].reshape(N, 7)
    grad = 0.5 * (s[:, 1::2] - s[:, 2::2]) / eps
    lap = ((s[:, 1::2] + s[:, 2::2]) - 2 * s[:, :1]).sum(-1) / eps2
    feature = out.reshape(N, 7, -1)[:, 0]
    # dh/dz of torch's Softplus(beta, threshold=20): exactly 1 where it returns z itself
    sig = torch.where(beta * z > 20, torch.ones_like(z), torch.sigmoid(beta * z))
    return s[:, 0], grad, feature, lap, dict(x01=x01, e=e, z=z, h=h, sig=sig, kernel_cells=kernel_cells)


def backward_fd(cache, table, lt, W1, b1, W2, b2, eps, eps2, n_active, g_out=None, g_sdf=None, g_grad=None, g_lap=None,
                kernel_cells=None):
    """upstream g_out [N,n_out], g_sdf [N], g_grad [N,3], g_lap [N] (None = 0) -> dict of gradients (W1, b1, W2, b2, table).
    kernel_cells (None: as the forward that made the cache): the kernels' fp32 cell fractions and fd_state values."""
    kernel_cells = cache.get('kernel_cells', False) if kernel_cells is None else kernel_cells
    if kernel_cells:
        eps, eps2 = _f32(eps), _f32(eps2)
    W1, W2 = W1.double(), W2.double()
    e, h, sig, x01 = cache['e'], cache['h'], cache['sig'], cache['x01']
    N, n_out = x01.shape[0] // 7, W2.shape[0]
    g = torch.zeros(N, 7, n_out, dtype=torch.float64)
    if g_out is not None:
        g[:, 0] += g_out.double()
    g0 = torch.zeros(N, 7, dtype=torch.float64)
    if g_sdf is not None:
        g0[:, 0] += g_sdf.double()
    if g_lap is not None:
        gl = g_lap.double() / eps2
        g0[:, 0] -= 6 * gl
        g0[:, 1:] += gl[:, None]
    if g_grad is not None:
        gg = 0.5 * g_grad.double() / eps
        g0[:, 1::2] += gg
        g0[:, 2::2] -= gg
    g[:, :, 0] += g0
    g = g.reshape(-1, n_out)
    zb = (g @ W2) * sig
    eb = zb @ W1
    dtable = torch.zeros_like(table.double().view(-1, 2))
    tab = table.double().view(-1, 2)
    for l in range(min(n_active, lt['n_levels'])):
        idx, w, _ = _level_terms(x01, tab, lt, l, kernel_cells)
        val = w[..., None] * eb[:, None, 3 + 2 * l: 5 + 2 * l]
        dtable.index_add_(0, idx.reshape(-1), val.reshape(-1, 2))
    return dict(W1=zb.t() @ e, b1=zb.sum(0), W2=g.t() @ h, b2=g.sum(0), table=dtable.reshape(-1))
