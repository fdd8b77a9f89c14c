"""One small invocation of every kernel, for compute-sanitizer (tools/sanitize.sh)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from stvo_pl_b200 import stereo_synth as SS, synth, types as T  # noqa: E402
from stvo_pl_b200.engine import Engine  # noqa: E402

eng = Engine(0)
cfg = T.kitti_config()
prev, curr, Tgt, cam = synth.make_batch("kitti", 3, n_pt=700, n_ls=180)
out = eng.track_batch(cam, cfg, prev, curr)
m = T.matched_from_frames(prev, curr, out["m12_pt"], out["m12_ls"])
eng.optimize_pose(cam, cfg, m)
cfg.solver_mode = 1
eng.track_batch(cam, cfg, prev, curr)
eng.gn_eval_stream(cam, cfg, m, Tgt, iters=1)
eng.match(prev.pdesc, curr.pdesc, 0.75)
# the streamed solver's long-list paths (several tiles per problem: records streamed, not resident) and an explicit list with flags
mb_hd, T_hd, cam_hd = synth.make_matched_batch("hd", 2)
eng.optimize_pose(cam_hd, T.kitti_config(), mb_hd)
q_cell, d1, t_cell, d2 = SS.make_stereo_points(500, 480, seed=1)
eng.match_grid_points([0, 500], q_cell, d1, [0, 480], t_cell, d2, T.PlGridWindow(10, 0, 0, 0), 0.75)
q_line, d1, t_line, t_dir, d2 = SS.make_stereo_lines(150, 160, seed=2)
eng.match_grid_lines([0, 150], q_line, d1, [0, 160], t_line, t_dir, d2, T.PlGridWindow(10, 0, 0, 0), 0.75, 0.75)
sc = T.default_stereo_config()
kp_l, octave, desc, kp_r, m12 = SS.make_lift_points(700, 650, seed=3)
eng.stereo_lift_points(cam, sc, [0, 700], kp_l, octave, desc, [0, 650], kp_r, m12)
seg_l, angle, octave, desc, seg_r, m12 = SS.make_lift_lines(300, 280, seed=4)
eng.stereo_lift_lines(cam, sc, [0, 300], seg_l, angle, octave, desc, [0, 280], seg_r, m12)
mc = T.default_stereo_match_config()
kp_l, octave, d1, kp_r, d2 = SS.make_stereo_frame_points(600, 580, seed=5)
eng.match_stereo_points(cam, mc, sc, [0, 600], kp_l, octave, d1, [0, 580], kp_r, d2)
seg_l, angle, octave, d1, seg_r, d2 = SS.make_stereo_frame_lines(250, 240, seed=6)
eng.match_stereo_lines(cam, mc, sc, [0, 250], seg_l, angle, octave, d1, [0, 240], seg_r, d2)
sp, scur, _, scam = SS.make_stereo_pairs(2, n_pt=500, n_ls=120, seed=7)
eng.track_stereo_batch(scam, T.kitti_config(), mc, sc, sp, scur)
sq, _, qcam = SS.make_stereo_sequence(4, n_pt=400, n_ls=90, seed=9)
eng.track_stereo_sequence(qcam, T.kitti_config(), mc, sc, sq)
pin = lambda d: {k: eng.pinned.copy(np.ascontiguousarray(v, T.STEREO_FEATURE_DTYPES[k])) for k, v in d.items()}
(pc, _k1), (cc, _k2) = T.stereo_features_as_c(pin(sp)), T.stereo_features_as_c(pin(scur))
ares, ans = eng.pinned.empty((2,), T.POSE_RESULT_DTYPE), eng.pinned.empty((2, 4), np.int32)
t1 = eng.track_stereo_batch_async(scam, T.kitti_config(), mc, sc, pc, cc, ares, ans)
t2 = eng.track_stereo_batch_async(scam, T.kitti_config(), mc, sc, pc, cc, ares, ans)
eng.wait(t1)
eng.wait(t2)
orb_imgs = np.stack([synth_img % 251 for synth_img in (np.arange(160 * 120, dtype=np.int64).reshape(120, 160) * 37,
                                                       np.arange(160 * 120, dtype=np.int64).reshape(120, 160) * 91)]).astype(np.uint8)
for st in (T.ORB_FAST_SCORE, T.ORB_HARRIS_SCORE):
    eng.orb_detect_and_compute_batch(T.default_orb_detect_config(300, score_type=st), orb_imgs, [10, 30])
print("sanitized run ok", int(out["results"]["good"].sum()))
