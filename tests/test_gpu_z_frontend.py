"""GPU parity of the training-batch front end (SURVEY 8f-3: nsr_gather_rays behind nsr_b200.rays.training_batch / image_batch) against
oracle/rays.py (numpy fp32 restatement of systems/nerf.py:33-91 + models/ray_utils.py, pinned to the reference's golden vectors).
Tolerance: origins, colours, masks exact (copies; the mask blend is three fp32 ops in the reference's order); directions 2e-7 absolute
(the order of the 3-term sums inside torch is not specified).

The n = 0 call at the end of the first test is an early return."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import rays as orays

D = torch.device('cuda:0')


def _dataset(seed, n_img=5, H=37, W=53, per_image_dirs=False, rows=3):
    rng = np.random.default_rng(seed)
    d = orays.get_ray_directions(W, H, 60.0, 61.0, W / 2, H / 2)
    if per_image_dirs:
        d = np.stack([d * np.float32(1 + 0.01 * i) for i in range(n_img)])
    c2w = np.zeros((n_img, rows, 4), np.float32)
    for i in range(n_img):
        q, _ = np.linalg.qr(rng.standard_normal((3, 3)))
        c2w[i, :3, :3], c2w[i, :3, 3] = q, rng.standard_normal(3) * 3
    if rows == 4:
        c2w[:, 3, 3] = 1
    images = rng.random((n_img, H, W, 4)).astype(np.float32)      # RGBA storage: only the first 3 channels are colours
    masks = (rng.random((n_img, H, W)) > 0.4).astype(np.float32)
    return d, c2w, images, masks


@pytest.mark.parametrize('per_image_dirs,rows,apply_mask', [(False, 3, False), (True, 4, True)])
def test_training_batch_matches_oracle(per_image_dirs, rows, apply_mask):
    from nsr_b200 import rays
    d, c2w, images, masks = _dataset(0, per_image_dirs=per_image_dirs, rows=rows)
    rng = np.random.default_rng(1)
    n = 4099
    idx, x, y = rng.integers(0, c2w.shape[0], n), rng.integers(0, d.shape[-2], n), rng.integers(0, d.shape[-3], n)
    bg = np.array([0.2, 0.5, 0.9], np.float32)
    ref_rays, ref_rgb, ref_fg = orays.training_batch(d, c2w, images, masks, idx, x, y, bg=bg, apply_mask=apply_mask)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(D)
    out = rays.training_batch(t(d), t(c2w), t(images), t(masks), t(idx), t(x), t(y), background_color=t(bg), apply_mask=apply_mask)
    got = {k: v.cpu().numpy() for k, v in out.items()}
    assert got['rays'].shape == (n, 6) and got['rgb'].shape == (n, 3) and got['fg_mask'].shape == (n,)
    np.testing.assert_array_equal(got['rays'][:, :3], ref_rays[:, :3])
    np.testing.assert_allclose(got['rays'][:, 3:], ref_rays[:, 3:], rtol=0, atol=2e-7)
    np.testing.assert_array_equal(got['fg_mask'], ref_fg)
    np.testing.assert_allclose(got['rgb'], ref_rgb, rtol=0, atol=1e-7)
    empty = rays.training_batch(t(d), t(c2w), t(images), t(masks), t(idx[:0]), t(x[:0]), t(y[:0]))
    assert empty['rays'].shape == (0, 6)


def test_image_batch_matches_oracle_and_the_reference_helpers():
    from nsr_b200 import rays
    d, c2w, images, masks = _dataset(2)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(D)
    out = rays.image_batch(t(d), t(c2w), 3, all_images=t(images), all_fg_masks=t(masks))
    ref = orays.image_batch(d, c2w, 3)
    np.testing.assert_array_equal(out['rays'][:, :3].cpu().numpy(), ref[:, :3])
    np.testing.assert_allclose(out['rays'][:, 3:].cpu().numpy(), ref[:, 3:], rtol=0, atol=2e-7)
    np.testing.assert_array_equal(out['rgb'].cpu().numpy(), images[3].reshape(-1, 4)[:, :3])
    np.testing.assert_array_equal(out['fg_mask'].cpu().numpy(), masks[3].reshape(-1))
    # the load-time torch helpers (reference signatures) agree with the kernel
    ro, rd = rays.get_rays(t(d), t(c2w)[3])
    np.testing.assert_allclose(torch.nn.functional.normalize(rd, dim=-1).cpu().numpy(), out['rays'][:, 3:].cpu().numpy(), atol=3e-7)
    with pytest.raises(IndexError):
        rays.image_batch(t(d), t(c2w), 5)
