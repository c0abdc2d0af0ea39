"""Deferred device error flags of the log-odds Octomap: two tracker flags raised before one sync are both reported, as an
input error, not as an exhausted block pool."""
import numpy as np
import pytest

import octo_logodds_reference as ref
from taichislam_b200 import synthetic as syn

pytestmark = pytest.mark.gpu

VS = 0.05
CAM = dict(fx=syn.FX / 4, fy=syn.FY / 4, cx=syn.CX / 4, cy=syn.CY / 4, width=160, height=120, step=2, max_range=3.0)


def test_two_tracker_flags_in_one_sync():
    import torch
    from taichislam_b200 import _capi as capi
    from taichislam_b200.octo_handle import OctoHandle
    dev = torch.device("cuda", torch.cuda.current_device())
    h = OctoHandle(256, 256, K=2, voxel_scale=VS, logodds=ref.params(), Kcam=syn.K_DEPTH, max_ray_length=5.0)
    h.integrate_points(np.array([[0.0, 0.3, 0.35]], np.float32), np.eye(3), np.zeros(3))   # the origin cell FREE
    h.travel_multi_update(0, np.zeros((1, 3), np.float32))
    h.sync()
    # torch in: neither call synchronises, so both flags are pending at the sync below
    h.view_gain_unknown(torch.zeros((1, 3), device=dev), 2.0 * torch.eye(3, device=dev)[None], CAM)   # leaves its window
    _, ln = h.travel_multi_path(torch.tensor([-1], dtype=torch.int32, device=dev), torch.zeros((1, 3), device=dev))
    with pytest.raises(capi.TslamError) as e:
        h.sync()
    assert e.value.code == capi.E_INVALID
    msg = str(e.value)
    assert "bitmap window" in msg and "source index" in msg, msg
    assert "pool" not in msg, msg
    assert int(ln[0]) == 0
    h.sync()                                                     # reported once
