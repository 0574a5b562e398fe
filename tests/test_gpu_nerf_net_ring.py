"""The network half of the split backward (nsr_nerf_field_bwd_net, also inside nsr_nerf_field_bwd_split) at row counts around multiples of
its work split, against the fp64 reference.  The kernel runs one CTA per SM (S = SM count) over 64-row tiles; the CTA's tiles alternate
between two chain groups and pass through a ring of three slots to the weight-gradient warpgroup.  64 S m +- 1 rows give CTAs m - 1, m or
m + 1 tiles for m = 1..4: a single tile, both groups, a full ring, and the first reuse of a slot by the other group; the last tile holds
one row or is one row short, and rows past the device count are NaN."""
import pytest

pytestmark = pytest.mark.gpu

from test_gpu_nerf_field_bwd import _check_forms, env  # noqa: F401  (env: the module fixture of the field backward tests)
from helpers import field_bwd_ref as fb


@pytest.mark.parametrize('m', [1, 2, 3, 4])
@pytest.mark.parametrize('delta', [-1, 1])
def test_net_ring_row_counts(env, m, delta):  # noqa: F811
    k = 64 * env.S * m + delta
    R = _check_forms(env, 'prod', env.inputs('prod', 270000), k, k + 100, 0.0, 'auto', forms=('F2', 'F3'))
    assert int(R['tie_rows'].sum()) <= max(1, fb.TIE_ROW_LIMIT * k)
