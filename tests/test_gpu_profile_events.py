"""derp_profile's event logs: while profiling is on, every brute-force sweep (plain or filtered) and every pingPongKernel
launch is counted and timed; re-enabling starts both logs and the ping-pong counters afresh; and a context destroyed
while profiling is on releases its events without an error."""
import pytest

from facebook360_dep_b200 import capi
from tests.parity_util import scene_inputs

pytestmark = pytest.mark.gpu


def test_profile_logs_sweeps_and_ping_pong(cuda):
    W, H = 96, 80
    rig, colors, _ = scene_inputs(num_cams=4, width=W, height=H, kind="RECTILINEAR", hfov_deg=120.0)
    ctx = capi.Context(cuda, capi.rig_descs(rig))
    ctx.level_begin(W, H)
    ctx.set_colors(colors)
    ctx.reproject(0)
    ctx.profile(True)
    for mode in (1, 2):  # the plain sweep, then the filtered one
        ctx.set_sweep_mode(mode)
        ctx.brute_force(0, num_depths=64)
    assert ctx.sweep_stats()[1] > 0, "the second sweep must have run filtered"
    ctx.ping_pong(0, iterations=3)

    ms, launches = ctx.get_profile()
    assert launches == 2 and ms > 0
    pp_ms, pp_launches, evals, _ = ctx.get_profile_ping_pong()
    assert pp_launches == 3 and pp_ms > 0 and evals > 0

    ctx.profile(True)
    assert ctx.get_profile() == (0.0, 0)
    assert ctx.get_profile_ping_pong()[:3] == (0.0, 0, 0)

    ctx.brute_force(0, num_depths=64)
    ctx.ping_pong(0)
    # derp_destroy returns nothing, so a leak is not observable here; what is checked is that destroying a context whose
    # logs hold events leaves the device usable: a fresh context profiles its own sweep and reports no stale launches
    ctx.close()
    ctx = capi.Context(cuda, capi.rig_descs(rig))
    ctx.level_begin(W, H)
    ctx.set_colors(colors)
    ctx.reproject(0)
    ctx.profile(True)
    ctx.brute_force(0, num_depths=64)
    ms, launches = ctx.get_profile()
    assert launches == 1 and ms > 0
    ctx.sync()
    ctx.close()
