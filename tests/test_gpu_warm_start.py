"""The warm start applied per body in chain order (k_build_rows leaves each chain entry's share, k_warm_start walks the chains; DESIGN.md
section 2.8): the momentum and the solver states after nb_setup_contact_constraints equal the CPU oracle bit for bit on settled piles, a
mixed box / sphere stack, a moving kinematic platform and a hub body; bodies without a contact, body 0 and kinematic bodies keep their rows
exactly; and nb_step, whose warm start runs straight into the sweeps, equals the staged calls step after step."""
import numpy as np
import pytest
import nudge_b200
from nudge_b200 import scenes
from tests.kinematic_ref import KinematicOracleSim, with_kinematic_ground
from tests.parity_util import Report, rows_by_contact, sync_oracle_from_gpu

pytestmark = pytest.mark.gpu


def _setup_parity(o, g, kinematic=(), free=False):
    """From the same state: collide ... setup on both; the momentum and warm-start states against the oracle, and the rows the warm start
    must leave alone (body 0, kinematic bodies, bodies in no contact) against the momentum before setup."""
    sync_oracle_from_gpu(o, g)
    o.collide(); g.collide()
    o.apply_gravity_damping(); g.apply_gravity_damping()
    g.download_bodies()
    before = g.momentum.copy()
    o.read_cached_impulses(); g.read_cached_impulses()
    o.setup_contact_constraints(); g.setup_contact_constraints()
    g.download_bodies(); g.download_contacts()
    n = g.counts().contacts
    assert n > 0 and g.counts().overflow == 0
    rep = Report("%s warm start" % o.scene.name)
    rep.eq("momentum after setup", o.momentum, g.momentum)
    gk = g.constraints_view()
    rep.eq("warm-start states", rows_by_contact(o.constraints_view(), n)["states"][gk["contact"].astype(np.int64)], gk["states"])
    bodies = g.contacts_view()["bodies"]
    moved = np.zeros(len(before), bool)
    moved[bodies["a"].astype(np.int64)] = True; moved[bodies["b"].astype(np.int64)] = True
    moved[0] = False; moved[list(kinematic)] = False
    if free:
        rep.check("bodies in no contact", (~moved[1:]).any())
    rep.eq("rows the warm start leaves alone", before[~moved], g.momentum[~moved])
    assert rep.ok, str(rep)


def _pair(scene, oracle=None):
    from oracle import pyoracle
    o = oracle or pyoracle.OracleSim(scene)
    g = nudge_b200.Sim(scene, contact_capacity=o.cap, debug=True)
    assert g.lut_model_exact(), "host CPU's rcpps/rsqrtps do not follow the LUT model: bit parity is not expected on this box"
    return o, g


@pytest.mark.parametrize("name", ["box_pile_8k", "box_sphere_stack", "falling"])
def test_warm_start_equals_oracle(name):
    s = {"box_pile_8k": lambda: scenes.box_drop(8000, iterations=8), "box_sphere_stack": lambda: scenes.mixed_stack(8190, iterations=16),
         "falling": lambda: scenes.demo_scene(300, 300, iterations=4, spread=8.0, height=14.0, seed=31)}[name]()
    o, g = _pair(s)
    for _ in range(300 if name != "falling" else 20):   # falling: the lowest bodies have landed, the rest are still in the air
        g.step()
    for _ in range(2):
        _setup_parity(o, g, free=name == "falling")
        g.apply_impulses(int(s.iterations)); g.update_cached_impulses(); g.write_cached_impulses(); g.advance()


def test_warm_start_equals_oracle_on_a_moving_kinematic_platform():
    """The pile on a kinematic ground that slides and turns (tests/kinematic_ref.with_kinematic_ground): its sides are read, never written."""
    base = scenes.box_drop(600, iterations=8, density_L=14.0, spacing=(2.2, 2.4, 2.2), rotate=True)
    s, k = with_kinematic_ground(base, (0.75, 0.0, 0.25), (0.0, 0.4, 0.0))
    o, g = _pair(s, KinematicOracleSim(s, contact_capacity=1 << 16))
    for _ in range(30):
        g.step()
    for _ in range(3):
        _setup_parity(o, g, kinematic=(k,))
        g.apply_impulses(int(s.iterations)); g.update_cached_impulses(); g.write_cached_impulses(); g.advance()


def test_warm_start_equals_oracle_on_a_hub_body():
    """hub_platform: 900 small boxes on one dynamic platform body, whose chain holds thousands of entries: k_warm_start walks it in one
    thread."""
    s = scenes.hub_platform(30, iterations=4)
    o, g = _pair(s)
    for _ in range(3):
        g.step()
    _setup_parity(o, g)


def _state(x):
    x.download_bodies(); x.download_cache()
    cv = x.cache_view()
    return b"".join(np.ascontiguousarray(a).tobytes() for a in (x.transforms, x.momentum, x.idle, cv["tags"], cv["features"], cv["data"]))


@pytest.mark.parametrize("name", ["box_drop", "hub"])
def test_step_equals_staged_calls(name):
    s = scenes.box_drop(3000, iterations=8) if name == "box_drop" else scenes.hub_platform(30, iterations=4)
    a, b = nudge_b200.Sim(s), nudge_b200.Sim(s)
    for i in range(30):
        a.step(); b.step_staged()
        assert _state(a) == _state(b), i
        assert a.counts().overflow == 0
