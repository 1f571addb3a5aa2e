"""The persistent conv kernel on grids where every CTA walks many work units."""
import pytest

from test_gpu_tcconv import test_merged_transposed_conv_phases_equal_separate_launches as _merged_equal_separate

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('b,c,cout,hw,split', [
    # ~2900 work units (4 phases x 2 channel tiles x 4 samples): each CTA crosses phase, channel-tile and sample boundaries
    (4, 256, 256, (96, 96), False),
])
def test_merged_phases_many_units_per_cta(b, c, cout, hw, split, monkeypatch):
    _merged_equal_separate(b, c, cout, hw, split, monkeypatch)
