"""State files (nb_save_state / nb_load_state, SURVEY.md section 8 f3) and the headless replay tool tools/nb_replay.cpp: a dumped state,
loaded into a fresh context or replayed by the CLI in another process, continues bit-identically; every file version is the documented
layout byte for byte, and a version-1 file loads the same whatever its undefined reserved words hold."""
import os, subprocess, tempfile
import numpy as np
import pytest
import nudge_b200
from nudge_b200 import scenes
from tests.gpu_util import STATE_HEADER, fnv1a, side_stream, state_file

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_state_roundtrip_and_headless_replay():
    import torch
    s = scenes.demo_scene(300, 300, iterations=8, spread=4.0, height=30.0)
    s.connections = np.zeros(3, scenes.PAIR32); s.connections["a"] = (1, 5, 9); s.connections["b"] = (2, 6, 10)
    side = torch.cuda.Stream()
    g = nudge_b200.Sim(s, stream=side.cuda_stream)
    for _ in range(60):
        g.step()
    d = tempfile.mkdtemp(prefix="nb_state_")
    p1, p2 = os.path.join(d, "a.bin"), os.path.join(d, "b.bin")
    g.save_state(p1)
    other = scenes.demo_scene(300, 300, iterations=8, seed=99); other.connections = np.zeros(3, scenes.PAIR32)   # different content, same capacities
    h = nudge_b200.Sim(other, stream=side.cuda_stream)
    h.load_state(p1)
    for _ in range(10):
        g.step(); h.step()
    g.download_bodies(); h.download_bodies(); g.download_cache(); h.download_cache()
    for name in ("transforms", "momentum", "idle"):
        assert getattr(g, name).tobytes() == getattr(h, name).tobytes(), name
    n = g.cache.count
    assert n == h.cache.count and g.cache_tags[:n].tobytes() == h.cache_tags[:n].tobytes() and g.cache_data[:n].tobytes() == h.cache_data[:n].tobytes()
    # the CLI, another process: same 10 steps from the same file
    exe = os.path.join(ROOT, "tools", "bin", "nb_replay")
    assert os.path.exists(exe), "tools/bin/nb_replay not built (nudge_b200/csrc/build.sh)"
    out = subprocess.run([exe, p1, "--steps", "10", "--iterations", "8", "--dump", p2], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    last = out.stdout.strip().splitlines()[-1].split()
    assert last[0] == "step" and last[1] == "9"
    assert int(last[last.index("xf") + 1], 16) == fnv1a(g.transforms.tobytes())
    assert int(last[last.index("contacts") + 1]) == g.counts().contacts
    k = nudge_b200.Sim(other, stream=side.cuda_stream)
    k.load_state(p2)
    k.download_bodies()
    assert k.transforms.tobytes() == g.transforms.tobytes() and k.momentum.tobytes() == g.momentum.tobytes() and k.idle.tobytes() == g.idle.tobytes()


def _tables_scene():
    s = scenes.demo_scene(120, 120, iterations=4, spread=3.0, height=12.0, seed=14)
    s.connections = np.zeros(3, scenes.PAIR32); s.connections["a"] = (1, 5, 9); s.connections["b"] = (2, 6, 10)
    return s


def _expected_file(g, version, reserved, **tables):
    """g's state file rebuilt from the layout: bodies and cache downloaded, colliders and connections as uploaded, plus `tables`."""
    g.download_bodies(); g.download_cache()
    n = g.cache.count
    sec = dict(transforms=g.transforms, properties=g.properties, momentum=g.momentum, idle=g.idle, box_tags=g.box_tags, box_data=g.box_data,
               box_transforms=g.box_transforms, sphere_tags=g.sphere_tags, sphere_data=g.sphere_data, sphere_transforms=g.sphere_transforms,
               connections=g.connections, cache_tags=g.cache_tags[:n], cache_features=g.cache_features[:n], cache_data=g.cache_data[:n], **tables)
    counts = (len(g.transforms), len(g.box_tags), len(g.sphere_tags), len(g.connections), n)
    return state_file(counts, {k: v.tobytes() for k, v in sec.items()}, version, reserved)


def test_every_version_is_the_documented_layout_and_undefined_reserved_words_are_ignored():
    from tests.sensor_ref import add_sensors
    side = side_stream()
    d = tempfile.mkdtemp(prefix="nb_state_layout_")
    plain = nudge_b200.Sim(_tables_scene(), stream=side)
    fs = _tables_scene()
    n = fs.n_colliders
    fs.collision_filters = np.zeros(n, scenes.FILTER)
    fs.collision_filters["category"] = 1 << (np.arange(n) % 3); fs.collision_filters["mask"] = 0xffff; fs.collision_filters["mask"][::7] = 5
    fs.filter_flags = scenes.FILTER_SKIP_CONNECTED
    filtered = nudge_b200.Sim(fs, stream=side)
    ss = add_sensors(_tables_scene(), zones=[((0.0, 1.0, 0.0), (3.0, 1.0, 3.0))], proximity=[4, 8])
    sensor = nudge_b200.Sim(ss, stream=side)
    sensor.upload_sensors(ss.sensors, max_pairs=4096)
    ks = _tables_scene()
    ks.kinematic = np.zeros(2, scenes.KINEMATIC); ks.kinematic["body"] = (7, 3); ks.kinematic["velocity"] = ((0.0, 0.5, 0.0), (0.25, 0.0, 0.0))
    kin = nudge_b200.Sim(ks, stream=side)
    for _ in range(20):
        for x in (plain, filtered, sensor, kin):
            x.step()
    cases = (("plain", plain, 1, (0,) * 8, {}),
             ("filtered", filtered, 2, (scenes.FILTER_SKIP_CONNECTED, 1) + (0,) * 6, dict(filter=fs.collision_filters)),
             ("sensor", sensor, 3, (0, 0, 1, 4096) + (0,) * 4, dict(sensor=(ss.sensors != 0).astype(np.uint8))),
             ("kinematic", kin, 4, (0, 0, 0, 0, 2, 0, 0, 0), dict(kinematic=np.array([3, 7], np.uint32))))
    for name, g, version, reserved, tables in cases:
        p = os.path.join(d, name + ".bin")
        g.save_state(p)
        assert open(p, "rb").read() == _expected_file(g, version, reserved, **tables), name
        assert g.cache.count > 0, name
    # a version-1 file whose reserved words claim every table: they are not defined in version 1, so the set and tables go
    raw = bytearray(open(os.path.join(d, "plain.bin"), "rb").read())
    h = list(STATE_HEADER.unpack_from(raw))
    h[8:] = (scenes.FILTER_SKIP_CONNECTED, 1, 1, 4096, 2, 9, 9, 9)
    STATE_HEADER.pack_into(raw, 0, *h)
    p = os.path.join(d, "v1_reserved.bin")
    open(p, "wb").write(raw)
    kin.load_state(p)
    for i in range(5):
        plain.step(); kin.step()
        plain.download_bodies(); kin.download_bodies()
        for f in ("transforms", "momentum", "idle"):
            assert getattr(plain, f).tobytes() == getattr(kin, f).tobytes(), (f, i)
