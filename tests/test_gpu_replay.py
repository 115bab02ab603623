"""The replay of a recorded drive on the GPU (urban_road_filter_b200/replay.py): every cloud it writes is byte for byte
what Detector.filtered_cloud2_packed packs on the device for the same message, every MarkerArray is urf_build_markers
on that scan's vertices with the topic's own ghostcount, golden fixture clouds replay to what the unmodified reference
published, the reference tie order reaches the replay, and two devices write the same bag as one."""
import numpy as np
import pytest
import torch

from urban_road_filter_b200 import FULL_ROI, api, make_params, rosbag
from urban_road_filter_b200.api import build_markers
from urban_road_filter_b200.replay import output_topics, replay
from urban_road_filter_b200.rosbag import BagReader, BagWriter, Header, PointCloud2, PointField, Time, cloud_format
from urban_road_filter_b200.synth import CLOUD2_LAYOUTS, drive_bag

from test_gpu_reference_ties import _dual_scan
from util import Golden, cloud2_records, compare_strips, golden_names

pytestmark = pytest.mark.gpu

SENSORS = [("/left_os1/os1_cloud_node/points", "C1", "ouster"), ("/right_os1/os1_cloud_node/points", "C1", "ouster"),
           ("/left_velodyne/velodyne_points", "C1", "velodyne"), ("/right_velodyne/velodyne_points", "C1", "velodyne")]


@pytest.fixture(scope="module", autouse=True)
def gpu():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"


def outputs(path):
    out = {}
    with BagReader(path) as r:
        for topic, _, t, d in r.messages():
            out.setdefault(topic, []).append((tuple(t), bytes(d)))
    return out


def check_against_packed(src, dst, prm, tie_order="input"):
    """Every output message of dst against filtered_cloud2_packed / build_markers for its input message of src."""
    out = outputs(dst)
    det = api.Detector(max_points=1 << 18, params=prm, tie_order=tie_order)
    ghost, seen, compared = {}, {k: 0 for k in out}, 0
    with BagReader(src) as r:
        for topic, _, t, data in r.messages():
            msg = rosbag.decode_cloud2(data)
            f = cloud_format(msg, topic)
            res, clouds = det.filtered_cloud2_packed(bytes(msg.data), msg.width * msg.height, *f)
            names = output_topics(topic)
            if res.status == 1:
                continue
            for k in ("road", "curb", "roi", "road_probably"):
                tm, d = out[names[k]][seen[names[k]]]
                seen[names[k]] += 1
                c = rosbag.decode_cloud2(d)
                assert tm == tuple(t) and c.header == msg.header and c.width == clouds[k].shape[0]
                assert bytes(c.data) == clouds[k].tobytes(), f"{topic} at {tuple(t)}: {k} cloud"
                compared += 1
            if res.n_vert > 2:
                strips, ghost[topic] = build_markers(prm, res.vert, ghost.get(topic, 0))
                tm, d = out[names["road_marker"]][seen[names["road_marker"]]]
                seen[names["road_marker"]] += 1
                ms = rosbag.decode_marker_array(d)
                assert tm == tuple(t) and len(ms) == len(strips)
                for m, (sid, action, red, pts) in zip(ms, strips):
                    assert (m.id, m.action, m.color[0]) == (sid, 2 if action == 2 else 0, 1.0 if red else 0.0)
                    assert np.array_equal(np.array(m.points, np.float64).reshape(-1, 3), pts)
    det.close()
    assert seen == {k: len(v) for k, v in out.items()}, "the replay wrote messages the packed path does not publish"
    return compared


@pytest.mark.parametrize("roi", ["default", "full"])
def test_gpu_replay_writes_the_packed_clouds_and_markers(tmp_path, roi):
    src = str(tmp_path / "drive.bag")
    drive_bag(src, SENSORS, 4, seed=11, distinct=3)
    prm = make_params(**(FULL_ROI if roi == "full" else {}))
    dst = str(tmp_path / "out.bag")
    rep = replay(src, dst, devices=(0,), slots=4, batch=3, params=prm)
    assert rep.scans == {t: 4 for t, _, _ in SENSORS}
    assert check_against_packed(src, dst, prm) == 4 * 4 * 4


def golden_bag(path, g, layout="ouster"):
    step, fields = CLOUD2_LAYOUTS[layout]
    offs = {name: off for name, off, _ in fields}
    pts = np.ascontiguousarray(g.cloud, np.float32)
    rec = cloud2_records(pts, step, offs["x"], offs["y"], offs["z"], offs["intensity"], seed=7)
    msg = PointCloud2(Header(1, Time(5, 0), "os1"), 1, pts.shape[0], [PointField(n, o, d, 1) for n, o, d in fields], False,
                      step, step * pts.shape[0], rec, True)
    with BagWriter(path) as w:
        w.write("/os1/points", rosbag.POINTCLOUD2, Time(5, 0), rosbag.encode_cloud2(msg))
    return pts


@pytest.mark.parametrize("name", [n for n in golden_names() if "ties" not in n and not n.startswith("c5")])
def test_gpu_replay_publishes_what_the_reference_published(tmp_path, name):
    """As tests/test_glue.py for the glue node: roi / road / curb / road_probably record for record and in order, and the
    road_marker strips (simplification off), against the reference's outputs for the fixture's cloud."""
    g = Golden(name)
    src, dst = str(tmp_path / "g.bag"), str(tmp_path / "out.bag")
    pts = golden_bag(src, g)
    replay(src, dst, devices=(0,), slots=2, batch=1, params=g.params(simple_poly_allow=0, poly_z_avg_allow=0))
    out = outputs(dst)
    if not g.published:
        assert out == {}
        return
    names = output_topics("/os1/points")

    def expect(idx):
        e = np.zeros((len(idx), 8), np.float32)
        e[:, :3], e[:, 3], e[:, 4] = pts[idx, :3], 1.0, pts[idx, 3]
        return e.tobytes()

    ids = dict(road=g.road_ids, curb=g.curb_ids, roi=np.flatnonzero(g.label >= 0), road_probably=g.prob_ids)
    for k, idx in ids.items():
        (tm, d), = out[names[k]]
        assert tm == (5, 0) and bytes(rosbag.decode_cloud2(d).data) == expect(np.asarray(idx, np.int64)), f"{name}: {k}"
    if g.markers_published:
        (tm, d), = out[names["road_marker"]]
        strips = [(m.id, m.action, int(m.color[0] == 1.0), np.array(m.points, np.float64).reshape(-1, 3))
                  for m in rosbag.decode_marker_array(d)]
        compare_strips(strips, g.strips_raw, name + " raw strips")
    else:
        assert names["road_marker"] not in out


def test_gpu_replay_in_the_reference_tie_order(tmp_path):
    """A dual-return clip, every ring tied: the replay's clouds are the packed output under the reference tie order."""
    pts = _dual_scan("C1", 3, False)
    prm = make_params(**FULL_ROI)
    src, dst = str(tmp_path / "dual.bag"), str(tmp_path / "out.bag")
    step, fields = CLOUD2_LAYOUTS["ouster"]
    rec = cloud2_records(pts, step, 0, 4, 8, 16, seed=3)
    with BagWriter(src) as w:
        for k in range(3):
            msg = PointCloud2(Header(k, Time(9, k), "os1"), 1, pts.shape[0], [PointField(n, o, d, 1) for n, o, d in fields],
                              False, step, step * pts.shape[0], rec, True)
            w.write("/dual", rosbag.POINTCLOUD2, Time(9, k), rosbag.encode_cloud2(msg))
    replay(src, dst, devices=(0,), slots=2, batch=2, params=prm, reference_tie_order=True)
    assert check_against_packed(src, dst, prm, tie_order="reference") == 3 * 4
    det = api.Detector(max_points=pts.shape[0], params=prm)           # the input order differs: the option did something
    _, plain = det.filtered_cloud2_packed(rec, pts.shape[0], 48, 0, 4, 8, 16)
    det.close()
    out = outputs(dst)
    mine = b"".join(bytes(rosbag.decode_cloud2(out[f"/dual/{k}"][0][1]).data) for k in ("road", "curb", "road_probably"))
    assert mine != b"".join(plain[k].tobytes() for k in ("road", "curb", "road_probably"))


def test_gpu_replay_on_two_devices_writes_the_same_bag(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU visible")
    src = str(tmp_path / "drive.bag")
    drive_bag(src, SENSORS, 6, seed=5, distinct=3)
    one, two = str(tmp_path / "one.bag"), str(tmp_path / "two.bag")
    replay(src, one, devices=(0,), slots=3, batch=2)
    replay(src, two, devices=(0, 1), slots=3, batch=2)
    assert open(one, "rb").read() == open(two, "rb").read()
