"""Host-side refusals of configurations that would silently compute the wrong scans: beam tables and a map LUT of different
theta_dis, stacked maps that disagree on theta_dis / eps / max_range, and a 24-bit packed scan block on a map whose ranges
reach the 32 m where the block clamps.  No GPU needed (the refusals come before any device work)."""
import os

import numpy as np
import pytest
import torch

CPU = torch.device('cpu')
MAPS = os.path.join(os.path.dirname(__file__), '..', 'f1tenth_gym_b200', 'maps')


@pytest.fixture(scope='module')
def f110():
    import f1tenth_gym_b200 as f
    return f


@pytest.fixture(scope='module')
def host(f110):
    return f110.maps.load_map(os.path.join(MAPS, 'example_map.yaml'), '.png')


def test_simulator_refuses_other_theta_dis(f110, host):
    m4000 = f110.DeviceMap(host, CPU, theta_dis=4000)
    sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, 2, 0, num_envs=3, device=CPU)
    with pytest.raises(ValueError, match='theta_dis'):
        sim.set_device_map(m4000)
    assert sim.map is None
    sim.set_device_map(f110.DeviceMap(host, CPU))
    sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, 2, 0, num_envs=3, device=CPU, theta_dis=4000)
    with pytest.raises(ValueError, match='theta_dis'):
        sim.set_device_map(f110.DeviceMap(host, CPU))
    sim.set_device_map(m4000)
    # the beam tables step through the map's LUT with the simulator's increment
    assert sim.beams.c.theta_index_increment == f110.maps.theta_index_increment(1080, 4.7, 4000)
    assert sim.map.c.theta_dis == 4000


def test_scan_simulator_refuses_other_theta_dis(f110, host):
    ss = f110.ScanSimulator2D(100, 4.7, theta_dis=32767, device=CPU)
    with pytest.raises(ValueError, match='theta_dis'):
        ss.set_device_map(f110.DeviceMap(host, CPU))
    assert ss.map is None
    ss.set_device_map(f110.DeviceMap(host, CPU, theta_dis=32767))
    with pytest.raises(ValueError, match='theta_dis'):
        f110.ScanSimulator2D(100, 4.7, device=CPU).set_device_map(ss.map)


@pytest.mark.parametrize('kw', [dict(theta_dis=4000), dict(eps=0.01), dict(max_range=40.0)])
def test_stack_refuses_mixed_scan_settings(f110, host, kw):
    a, b = f110.DeviceMap(host, CPU), f110.DeviceMap(host, CPU, **kw)
    with pytest.raises(ValueError, match=list(kw)[0]):
        f110.DeviceMap.stack([a, b])
    st = f110.DeviceMap.stack([b, f110.DeviceMap(host, CPU, **kw)])
    k, v = list(kw.items())[0]
    assert getattr(st.c, k) == v and st.c.num_layers == 2


@pytest.mark.parametrize('max_range,noise', [(40.0, 0.0), (32.0, 0.0), (30.0, 0.25)])
def test_packed_scans_refuse_ranges_from_32m(f110, host, max_range, noise):
    """f110_pack_scans_u24 clamps at 32 m - 2^-19: make_host_pipeline(packed_scans=True) refuses a map whose max_range plus
    8 sigma of the scan noise reaches 32 m (before it allocates anything on the device)."""
    sim = f110.Simulator(f110.maps.DEFAULT_PARAMS, 1, 0, num_envs=2, device=CPU, noise_std=noise)
    sim.set_device_map(f110.DeviceMap(host, CPU, max_range=max_range))
    with pytest.raises(ValueError, match='packed_scans'):
        sim.make_host_pipeline(packed_scans=True)


def test_packed_scans_limit_value(f110):
    from f1tenth_gym_b200 import simulator
    assert simulator.PACKED_RANGE_LIMIT == 2.0 ** 24 * 2.0 ** -19
    # the largest code decodes to just below the limit
    buf = np.array([[255, 255, 255]], dtype=np.uint8)
    assert f110.Simulator.unpack_scans_u24(buf)[0] == np.float32(32.0 - 2.0 ** -19)
