"""Hand-derived forward/backward of the NeuS SDF field (VolumeSDF.forward with grad_type='analytic',
models/geometry.py:158-180; encoding = CompositeEncoding[2x-1 | HashGrid] network_utils.py:68-79; network = VanillaMLP with one
hidden layer and Softplus(beta=100), network_utils.py:95-139) -- CPU restatement of what the fused CUDA kernels compute, in
plain torch WITHOUT autograd.  tests/test_oracle_kat.py checks it against autograd (incl. the second-order terms the eikonal
loss needs); tests/helpers/neus_field_ref.py restates it with per-entry error bounds for the kernel tests.

Notation (per sample): e = [2 x01 - 1 (3) | hash(x01) (LF)];  z = W1 e + b1;  h = softplus_beta(z);  s = sigmoid(beta z) = dh/dz
out = W2 h + b2 (sdf = out_0);  u = s * W2[0];  q = W1^T u;  grad_world = (2 q_xyz + J^T q_hash) / (2 r),  J = d hash / d x01.
Backward for upstream (g_out [13], g_grad [3]):
  gx = g_grad / (2r);  qb = [2 gx | J gx];  ub = W1 qb;  zb = W2^T g_out * s + (ub * W2[0]) * beta s (1 - s);  eb = W1^T zb
  dW1 = u (x) qb + zb (x) e;  db1 = zb;  dW2 = g_out (x) h  (+ row 0: ub * s);  db2 = g_out
  dtable[corner c of level l] += w_c * eb_l + q_l * scale_l * (dw_c/dx . gx)
"""
import torch

from . import hashgrid


def x01_f32(points, radius):
    """the kernels' normalised position fp32(fp32(p + r) * fp32(1 / (2 r))): exactly the value their cell rule sees"""
    r = torch.tensor(radius, dtype=torch.float32)
    return (points.float() + r) * (1.0 / (2.0 * r))


def _level_terms(x01, table, lt, l, f32_frac=False):
    """cells / weights / derivative weights of level l: idx [N,8], w [N,8], dw [N,8,3] (d w_c / d x01, scale included).
    f32_frac: the fraction is the kernels' fp32 pos - floor(pos) (exact given pos) instead of the unrounded fp64 one."""
    scale = float(lt['scale'][l])
    pos32 = hashgrid.fma_f32(x01.float(), torch.tensor(scale, dtype=torch.float32), torch.tensor(0.5))
    cell = torch.floor(pos32)
    frac = (pos32.double() if f32_frac else x01.double() * scale + 0.5) - cell.double()
    ci = cell.to(torch.int64)
    res, size, dense, off = int(lt['res'][l]), int(lt['size'][l]), bool(lt['dense'][l]), int(lt['offset'][l])
    idx, w, dw = [], [], []
    for c in range(8):
        b = [(c >> a) & 1 for a in range(3)]
        f = [frac[:, a] if b[a] else 1 - frac[:, a] for a in range(3)]
        sg = [1.0 if b[a] else -1.0 for a in range(3)]
        w.append(f[0] * f[1] * f[2])
        dw.append(torch.stack([sg[0] * f[1] * f[2], f[0] * sg[1] * f[2], f[0] * f[1] * sg[2]], -1) * scale)
        idx.append(hashgrid.corner_index(ci[:, 0] + b[0], ci[:, 1] + b[1], ci[:, 2] + b[2], res, size, dense) + off)
    return torch.stack(idx, 1), torch.stack(w, 1), torch.stack(dw, 1)


def forward(points, table, lt, W1, b1, W2, b2, radius, beta=100.0, kernel_cells=False):
    """-> sdf [N], grad_world [N,3], feature [N,n_out], cache.
    kernel_cells: take x01 and the cell fractions as the kernels compute them in fp32 (x01_f32, then fp32 pos - floor(pos)), so that
    every level picks the same cell as the kernels, even for samples one ulp from a cell face; the rest stays fp64."""
    x01 = x01_f32(points, radius).double() if kernel_cells else (points.double() + radius) / (2 * radius)
    tab = table.double().view(-1, 2)
    L = lt['n_levels']
    feats, J = [], []
    for l in range(L):
        idx, w, dw = _level_terms(x01, tab, lt, l, kernel_cells)
        v = tab[idx]                                     # [N,8,2]
        feats.append((w[..., None] * v).sum(1))          # [N,2]
        J.append(torch.einsum('ncd,ncf->nfd', dw, v))    # [N,2,3]
    e = torch.cat([x01 * 2 - 1] + feats, -1)             # [N, 3+2L]
    J = torch.cat(J, 1)                                  # [N, 2L, 3]
    z = e @ W1.double().t() + b1.double()
    h = torch.nn.functional.softplus(z, beta=beta)
    s = torch.sigmoid(beta * z)
    out = h @ W2.double().t() + b2.double()
    u = s * W2.double()[0]
    q = u @ W1.double()                                  # [N, 3+2L]
    g01 = 2 * q[:, :3] + torch.einsum('nfd,nf->nd', J, q[:, 3:])
    return out[:, 0], g01 / (2 * radius), out, dict(x01=x01, e=e, J=J, z=z, h=h, s=s, u=u, q=q, kernel_cells=kernel_cells)


def backward(cache, table, lt, W1, b1, W2, b2, radius, g_out, g_grad, beta=100.0):
    """g_out [N,n_out] (dL/d out, sdf in slot 0), g_grad [N,3] (dL/d grad_world) -> dict of gradients."""
    W1, W2 = W1.double(), W2.double()
    e, J, s, h, u, q = cache['e'], cache['J'], cache['s'], cache['h'], cache['u'], cache['q']
    gx = g_grad.double() / (2 * radius)
    qb = torch.cat([2 * gx, torch.einsum('nfd,nd->nf', J, gx)], -1)
    ub = qb @ W1.t()
    zb = (g_out.double() @ W2) * s + (ub * W2[0]) * beta * s * (1 - s)
    eb = zb @ W1
    dW1 = u.t() @ qb + zb.t() @ e
    dW2 = g_out.double().t() @ h
    dW2[0] += (ub * s).sum(0)
    dtable = torch.zeros_like(table.double().view(-1, 2))
    x01 = cache['x01']
    tab = table.double().view(-1, 2)
    for l in range(lt['n_levels']):
        idx, w, dw = _level_terms(x01, tab, lt, l, cache.get('kernel_cells', False))
        ebl = eb[:, 3 + 2 * l: 5 + 2 * l]                # [N,2]
        ql = q[:, 3 + 2 * l: 5 + 2 * l]
        coef = torch.einsum('ncd,nd->nc', dw, gx)        # [N,8]
        val = w[..., None] * ebl[:, None, :] + coef[..., None] * ql[:, None, :]
        dtable.index_add_(0, idx.reshape(-1), val.reshape(-1, 2))
    return dict(W1=dW1, b1=zb.sum(0), W2=dW2, b2=g_out.double().sum(0), table=dtable.reshape(-1))
