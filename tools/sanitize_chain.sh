export TLOAM_B200_NO_GRAPH=1
cat > /tmp/seg_one.py <<PY
import sys; sys.path.insert(0, ".")
import numpy as np, tloam_b200
from tloam_b200 import synth
r = tloam_b200.LocalRegistration()
scan = synth.raw_scan(n_az=300)
o = r.segment_scan(scan, ring_min_num=16, dcvc=dict(min_seg=20))
print("segment_scan", {k: len(v) for k, v in o.items()})
big = np.random.default_rng(0).uniform(-40, 40, (200000, 3)) * np.array([1, 1, 0.05])
r.set_input_target([big[:5000].copy(), big[:20000].copy(), big, big[:90000].copy()])       # pageable: staged by the library
print("knn", r.knn(2, big[:100], 0.3, 5)[2].sum())
r.close()
PY
cat > /tmp/process_one.py <<PY
import sys; sys.path.insert(0, ".")
import numpy as np, tloam_b200
from tloam_b200 import synth
fe = dict(cvr_submap=0.005, cvr_scan=0.01)
r = tloam_b200.LocalRegistration()
r.enable_global_map()
scan = synth.raw_scan(n_az=300)
print("process_raw_scan", r.process_raw_scan(scan, ring_min_num=16, dcvc=dict(min_seg=20), feature=fe))
r.submap_init_frame()
T = synth.se3_exp([0.3, 0.02, 0, 0, 0, 0.004])
Ti = np.linalg.inv(T)
print("process_raw_scan", r.process_raw_scan(np.ascontiguousarray(scan @ Ti[:3, :3].T + Ti[:3, 3]), ring_min_num=16, dcvc=dict(min_seg=20), feature=fe))
r.scan_matching_predicted_async()
r.submap_update_frame_chained()
r.global_map_append_frame()
print("pose", r.get_result()[:3, 3])
r.global_map_append(np.vstack([scan, np.full((10, 3), np.nan)]), T)
print("global map", r.global_map_size(), len(r.registered_scan()))
inten = np.random.default_rng(0).uniform(0, 255, len(scan) + 10)
r.global_map_append(np.vstack([scan, np.full((10, 3), np.nan)]), T, intensity=inten)       # libtloam_b200_gmi.so
r.reset_global_map()
r.global_map_append(np.vstack([scan, np.full((10, 3), np.nan)]), T, intensity=inten)
r.global_map_append(scan, T)                                                                # clears the channel
r.global_map_append(np.vstack([scan, np.full((10, 3), np.nan)]), None, intensity=inten)
print("global map intensity", r.global_map_size(), r.global_map_has_intensity())
r.reset_global_map()
r.global_map_append(scan, T, intensity=inten[:len(scan)])
print("intensity", r.global_map_intensity()[:3])
# packed scans (libtloam_b200_unpack.so): a 22-byte velodyne XYZIRT message and a KITTI (n, 4) scan
dt = np.dtype(dict(names=["x", "y", "z", "intensity", "ring", "time"], formats=["<f4"] * 4 + ["<u2", "<f4"], offsets=[0, 4, 8, 12, 16, 18], itemsize=22))
msg = np.zeros(len(scan) + 10, dt)
f = np.vstack([scan, np.full((10, 3), np.nan)]).astype(np.float32)
msg["x"], msg["y"], msg["z"], msg["intensity"] = f[:, 0], f[:, 1], f[:, 2], inten.astype(np.float32)
print("segment_raw_scan_packed", {k: len(v) for k, v in r.segment_raw_scan_packed(msg, ring_min_num=16, dcvc=dict(min_seg=20)).items()})
print("process_raw_scan_packed", r.process_raw_scan_packed(msg, ring_min_num=16, dcvc=dict(min_seg=20), feature=fe))
r.global_map_append_frame(T)                                                                # the packed intensity, on the device
r.global_map_append_packed(np.ascontiguousarray(np.column_stack([f, inten.astype(np.float32)])), T)
r.global_map_append_packed(np.ascontiguousarray(f[:333]), None)
print("packed", r.global_map_size(), r.global_map_has_intensity())
r.close()
PY
for tool in memcheck racecheck; do
  echo "== $tool: tloam_b200_segment_scan + pageable staging (set_target of a 4.8 MB cloud)"
  timeout 600 compute-sanitizer --tool $tool --print-limit 5 python /tmp/seg_one.py 2>&1 | tail -4
  echo "== $tool: tloam_b200_process_raw_scan -> submap_init_frame -> scan_match_predicted_async -> submap_update_frame_chained -> global_map_append_frame_chained, global_map_append (with and without intensity), the packed-scan calls"
  timeout 600 compute-sanitizer --tool $tool --print-limit 5 python /tmp/process_one.py 2>&1 | tail -4
done
