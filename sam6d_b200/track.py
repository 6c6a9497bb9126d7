"""Object tracking through an RGB-D sequence (not in the reference): detect once with SAM6D.detect_objects, then follow each
object's pose from frame to frame with depth alone, and detect again only to start or recover a track.

    from sam6d_b200.track import Tracker
    objs = sam6d.onboard_objects(meshes, obj_ids=[1, 5])
    tracker = Tracker(sam6d, objs, meshes)                 # the same numpy meshes (mm), in the same order
    for rgb, depth in frames:
        res = tracker(rgb, depth, cam_K, depth_scale)      # res.R (O,3,3), res.t (O,3) metres; res.state; res.records

A tracked frame renders every live object at its previous pose (render.render, one call), selects each object's observed
points on the device (ops.track_points: the rendered silhouette dilated by margin_px, positive depth, a sphere of gate_scale x
the object's radius about its centroid), and refines the pose by point-to-plane ICP (ops.icp_refine) from the previous pose.
A track whose ICP ends with fewer than min_inlier_fraction of the points as inliers, or above max_rms_m, is lost.  Detection
runs on the first frame, on the frame after a track was lost, and when redetect_interval frames have passed without one; an
object with no live track starts from its highest-scoring PEM instance.  One track per object.  The defaults are not tuned on
real video, and whether tracking keeps the per-frame pipeline's accuracy on real sequences is unverified."""
import time
from types import SimpleNamespace

import numpy as np
import torch

from . import meshio, ops, pipeline, render
from .cli import pem_run_inference_custom as pem_cli

TRACKED, DETECTED, ABSENT = "tracked", "detected", "absent"


class Tracker:
    """one track per object of `objects` (an ObjectSet of `sam6d`).  meshes: the numpy meshes in mm passed to onboard_objects,
    in the same order (meshio.Mesh or PLY paths); they are uploaded once for rendering, and the ICP
    samples and normals come from pipeline.icp_model, whatever icp_iters sam6d has.  Parameters (defaults not tuned on real
    video): track_icp_iters ICP iterations per tracked frame; margin_px the silhouette dilation in pixels; gate_scale the gate
    radius over the object's radius about its model-point centroid; min_inlier_fraction and max_rms_m the loss rule;
    redetect_interval the frames after which detection runs again to pick up objects not yet found."""

    def __init__(self, sam6d, objects, meshes, track_icp_iters: int = 10, margin_px: int = 16, gate_scale: float = 1.5,
                 min_inlier_fraction: float = 0.5, max_rms_m: float = 0.005, redetect_interval: int = 30):
        meshes = [meshio.load_ply_mesh(m) if isinstance(m, str) else m for m in meshes]
        O = len(objects.obj_ids)
        if len(meshes) != O:
            raise ValueError(f"Tracker: {len(meshes)} meshes for {O} objects")
        if int(track_icp_iters) < 1 or int(margin_px) < 0 or not gate_scale > 0 or int(redetect_interval) < 1:
            raise ValueError("Tracker: track_icp_iters >= 1, margin_px >= 0, gate_scale > 0 and redetect_interval >= 1 are required")
        self.sam6d, self.objects = sam6d, objects
        self.track_icp_iters, self.margin_px, self.gate_scale = int(track_icp_iters), int(margin_px), float(gate_scale)
        self.min_inlier_fraction, self.max_rms_m, self.redetect_interval = float(min_inlier_fraction), float(max_rms_m), int(redetect_interval)
        self.n_points = pem_cli.TEST_DATASET["n_sample_observed_point"]
        dev = self.device = torch.device(sam6d.device)
        self.meshes = [render.upload(meshio.Mesh(vertices=m.vertices, faces=m.faces), dev) for m in meshes]
        self.icp = pipeline.icp_tensors(*(np.stack(a) for a in zip(*[pipeline.icp_model(m.vertices, m.faces) for m in meshes])), dev)
        mp = torch.from_numpy(np.ascontiguousarray(objects.model_points_m, dtype=np.float32)).to(dev)
        self.icp_radius = mp.norm(dim=2).amax(dim=1).contiguous()                       # as pipeline.icp_refine_out
        mp64 = np.asarray(objects.model_points_m, np.float64)
        centroid = mp64.mean(axis=1)
        self.centroid = torch.from_numpy(centroid.astype(np.float32)).to(dev)
        self.gate_radius = torch.from_numpy((self.gate_scale * np.linalg.norm(mp64 - centroid[:, None], axis=2).max(axis=1))
                                            .astype(np.float32)).to(dev)
        self.reset()

    def reset(self):
        """drop every track; the next frame runs detection"""
        O = len(self.objects.obj_ids)
        self.R = torch.full((O, 3, 3), float("nan"), device=self.device)
        self.t = torch.full((O, 3), float("nan"), device=self.device)
        self.live = np.zeros(O, bool)
        self.score = np.zeros(O)
        self.frames_tracked = np.zeros(O, np.int64)
        self._since_detection = None            # None: no detection since construction or reset()
        self._lost = False

    def start(self, o: int, R, t, score: float = 1.0):
        """seed object o's track at pose R (3,3), t (3,) in metres"""
        self.R[o] = torch.as_tensor(R, dtype=torch.float32, device=self.device).reshape(3, 3)
        self.t[o] = torch.as_tensor(t, dtype=torch.float32, device=self.device).reshape(3)
        self.live[o], self.score[o], self.frames_tracked[o] = True, float(score), 0

    def detection_due(self) -> bool:
        return self._since_detection is None or self._lost or self._since_detection >= self.redetect_interval

    def __call__(self, rgb_u8: np.ndarray, depth_raw: np.ndarray, cam_K, depth_scale):
        """one frame: rgb (H,W,3) u8, depth (H,W) raw u16, cam_K (9 values), depth_scale as camera.json holds them ->
        SimpleNamespace(R (O,3,3), t (O,3) metres on the device, NaN rows for objects with no track; state (O) "tracked",
        "detected" or "absent"; inliers (O) and rms (O) metres of the tracking ICP (-1 and NaN where it did not run); records,
        one per live object with pem_records' keys plus track and frames_tracked; detection, detect_objects' result when
        detection ran on this frame, else None)"""
        t0 = time.time()
        O = len(self.objects.obj_ids)
        H, W = depth_raw.shape
        K = np.asarray(cam_K, np.float64).reshape(3, 3)
        state = [ABSENT] * O
        inliers, rms = np.full(O, -1, np.int64), np.full(O, np.nan)
        live = np.flatnonzero(self.live)
        cand = None
        if len(live):
            cand = self._track(live, np.ascontiguousarray(depth_raw, dtype=np.uint16), K, depth_scale, H, W, inliers, rms)
            for o in live:
                if self.live[o]:
                    state[o] = TRACKED
                    self.frames_tracked[o] += 1
        lost = len(live) > int(self.live[live].sum())
        detection, started = None, {}
        if self.detection_due():
            detection = self.sam6d.detect_objects(rgb_u8, depth_raw, cam_K, depth_scale, self.objects)
            self._since_detection = 0
            started = self._start_from(detection, state)
        else:
            self._since_detection += 1
        self._lost = lost
        records = self._records(state, started, cand, live, (H, W), time.time() - t0)
        return SimpleNamespace(R=self.R.clone(), t=self.t.clone(), state=state, inliers=inliers, rms=rms, records=records,
                               detection=detection)

    def _track(self, live, depth_raw, K, depth_scale, H, W, inliers, rms):
        """render, select points and refine every live object; drop the tracks the loss rule rejects -> the candidate masks"""
        idx = torch.from_numpy(live).to(self.device)
        R, t = self.R[idx].contiguous(), self.t[idx].contiguous()
        poses = torch.zeros(len(live), 1, 4, 4, device=self.device)
        poses[:, 0, :3, :3] = R
        poses[:, 0, :3, 3] = t * 1000.0                                                   # the meshes are in mm
        poses[:, 0, 3, 3] = 1.0
        rdepth = render.render([self.meshes[o] for o in live], poses, K, H, W)["depth"][:, 0].contiguous()
        centre = (torch.einsum("lij,lj->li", R, self.centroid[idx]) + t).contiguous()
        depth_d = torch.from_numpy(depth_raw).to(self.device)
        pts, _, cand = ops.track_points(rdepth, depth_d, depth_scale, K, centre, self.gate_radius[idx].contiguous(), self.margin_px,
                                        self.n_points)
        R1, t1, inl, err, _ = ops.icp_refine(R, t, pts, self.icp[0], self.icp[1], idx.to(torch.int32), self.icp_radius[idx].contiguous(),
                                             self.track_icp_iters)
        inl, err = inl.cpu().numpy(), err.cpu().numpy()
        self.R[idx], self.t[idx] = R1, t1
        for j, o in enumerate(live):
            inliers[o], rms[o] = inl[j], err[j]
            if inl[j] < self.min_inlier_fraction * self.n_points or err[j] > self.max_rms_m:
                self.live[o] = False
                self.R[o], self.t[o] = float("nan"), float("nan")
        return cand

    def _start_from(self, det, state):
        """start each object with no live track from its highest-scoring PEM instance of detect_objects' result -> {object:
        the PEM record that started it}"""
        frame, started = det.frame, {}
        if frame is None or frame.out is None or not det.pem:
            return started
        obj, scores = np.asarray(frame.obj), np.asarray(frame.pose_scores)
        for o in range(len(state)):
            rows = np.flatnonzero(obj == o)
            if self.live[o] or not len(rows):
                continue
            best = int(rows[np.argmax(scores[rows])])                                   # the first of equal scores
            self.R[o], self.t[o] = det.R[best], det.t[best]
            self.live[o], self.score[o], self.frames_tracked[o] = True, float(scores[best]), 0
            started[o] = dict(det.pem[best])
            state[o] = DETECTED
        return started

    def _records(self, state, started, cand, live, hw, runtime):
        """one record per live object: a detected object's PEM record, a tracked object's pose with the bbox and RLE of its
        candidate pixels; each with track (the state) and frames_tracked"""
        O = len(state)
        R, t = self.R.cpu().numpy(), self.t.cpu().numpy() * 1000.0
        rec = [None] * O
        tracked = [o for o in range(O) if state[o] == TRACKED]
        if tracked:
            rows = [int(np.flatnonzero(live == o)[0]) for o in tracked]
            m = cand[torch.tensor(rows, device=cand.device)]
            cum, off = ops.mask_rle(m.float().contiguous())
            counts = pipeline.rle_counts(cum.cpu().numpy(), off.cpu().numpy())
            ys, xs = m.any(dim=2).cpu().numpy(), m.any(dim=1).cpu().numpy()
            for j, o in enumerate(tracked):
                y, x = np.flatnonzero(ys[j]), np.flatnonzero(xs[j])
                bbox = [int(x[0]), int(y[0]), int(x[-1] + 1 - x[0]), int(y[-1] + 1 - y[0])] if len(x) else [0, 0, 0, 0]
                rec[o] = dict(scene_id=0, image_id=0, category_id=int(self.objects.obj_ids[o]), bbox=bbox, score=float(self.score[o]),
                              time=float(runtime), segmentation={"counts": counts[j], "size": [int(hw[0]), int(hw[1])]})
        for o in range(O):
            if state[o] == DETECTED:
                rec[o] = started[o]
            if rec[o] is not None:
                rec[o].update(R=R[o].tolist(), t=t[o].tolist(), track=state[o], frames_tracked=int(self.frames_tracked[o]))
        return [r for r in rec if r is not None]
