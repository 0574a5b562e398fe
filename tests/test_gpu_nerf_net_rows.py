"""The network half of the split backward (nsr_nerf_field_bwd_net, also inside nsr_nerf_field_bwd_split) at row counts around one
warpgroup tile, against the fp64 reference.  Each chain warpgroup runs the ten GEMMs of a 64-row tile as register-A wgmma over its four
warps: 1, 63, 64 and 65 rows give a tile with one live row, a tile one row short, exactly one full tile, and a full tile plus a one-row
tile on a second CTA; 2 * 64 S + 37 rows (S = SM count) give every CTA full tiles on two chain groups and the first CTA a partial tile
on its third.
d(encoding) and the five weight gradients are checked entry by entry; rows past the device count are NaN."""
import pytest

pytestmark = pytest.mark.gpu

from test_gpu_nerf_field_bwd import _check_forms, env  # noqa: F401  (env: the module fixture of the field backward tests)
from helpers import field_bwd_ref as fb


@pytest.mark.parametrize('rows', ['1', '63', '64', '65', '2x64S+37'])
def test_net_rows_match_reference(env, rows):  # noqa: F811
    k = 2 * 64 * env.S + 37 if rows == '2x64S+37' else int(rows)
    R = _check_forms(env, 'prod', env.inputs('prod', 270000), k, k + 100, 0.0, 'auto', forms=('F2', 'F3'))
    assert int(R['tie_rows'].sum()) <= max(1, fb.TIE_ROW_LIMIT * k)
