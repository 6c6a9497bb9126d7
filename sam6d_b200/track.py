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
object with no live track starts from its highest-scoring PEM instance.  The defaults are not tuned on real video, and
whether tracking keeps the per-frame pipeline's accuracy on real sequences is unverified.

With max_instances = I > 1 an object may have up to I tracks, for scenes with several copies of one object.  Each pixel then
goes to at most one track (ops.track_points_scene: the track rendered in front there, else the one nearest its gate centre
relative to its radius), so tracks of overlapping copies do not share points.  After the ICP a track whose centroid lies within
assoc_scale x the object's radius of an older track's of the same object is dropped as a duplicate (a loss: detection runs on
the next frame), and detection starts further tracks of an object from its PEM instances that score at least start_score
and lie farther than that from every track of the object.  start_score and assoc_scale are not tuned on real video, and the
centroid test cannot tell apart copies whose centroids lie closer than assoc_scale x the radius, such as flat objects
stacked on one another."""
import time
from types import SimpleNamespace

import numpy as np
import torch

from . import meshio, ops, pipeline, render
from .cli import pem_run_inference_custom as pem_cli

TRACKED, DETECTED, ABSENT = "tracked", "detected", "absent"


class Tracker:
    """up to max_instances tracks per object of `objects` (an ObjectSet of `sam6d`).  meshes: the numpy meshes in mm passed
    to onboard_objects, in the same order (meshio.Mesh or PLY paths); they are uploaded once for rendering, and the ICP
    samples and normals come from pipeline.build_pose_inputs, whatever icp_iters sam6d has.  Parameters (defaults not tuned
    on real video): track_icp_iters ICP iterations per tracked frame; margin_px the silhouette dilation in pixels; gate_scale
    the gate radius over the object's radius about its model-point centroid; min_inlier_fraction and max_rms_m the loss rule;
    redetect_interval the frames after which detection runs again to pick up objects not yet found; max_instances I the
    tracks per object, start_score the least PEM score that starts an object's second and later tracks, assoc_scale the
    centroid distance, over the object's radius about its centroid, within which two tracks of one object are one copy.

    Tracks live in O x I slots, slot o I + k belonging to object o (with I = 1, slot o is object o); res.R, t, state, inliers,
    rms, track_id and obj are indexed by slot.  Track ids count up from 0 after construction or reset() and are never reused."""

    def __init__(self, sam6d, objects, meshes, track_icp_iters: int = 10, margin_px: int = 16, gate_scale: float = 1.5,
                 min_inlier_fraction: float = 0.5, max_rms_m: float = 0.005, redetect_interval: int = 30, max_instances: int = 1,
                 start_score: float = 0.3, assoc_scale: float = 0.5):
        meshes = [meshio.load_ply_mesh(m) if isinstance(m, str) else m for m in meshes]
        O = len(objects.obj_ids)
        if len(meshes) != O:
            raise ValueError(f"Tracker: {len(meshes)} meshes for {O} objects")
        if int(track_icp_iters) < 1 or int(margin_px) < 0 or not gate_scale > 0 or int(redetect_interval) < 1:
            raise ValueError("Tracker: track_icp_iters >= 1, margin_px >= 0, gate_scale > 0 and redetect_interval >= 1 are required")
        if int(max_instances) < 1 or not assoc_scale >= 0:
            raise ValueError("Tracker: max_instances >= 1 and assoc_scale >= 0 are required")
        self.sam6d, self.objects = sam6d, objects
        self.track_icp_iters, self.margin_px, self.gate_scale = int(track_icp_iters), int(margin_px), float(gate_scale)
        self.min_inlier_fraction, self.max_rms_m, self.redetect_interval = float(min_inlier_fraction), float(max_rms_m), int(redetect_interval)
        self.max_instances, self.start_score, self.assoc_scale = int(max_instances), float(start_score), float(assoc_scale)
        self.obj = np.repeat(np.arange(O), self.max_instances)                         # slot -> object
        self.n_points = pem_cli.TEST_DATASET["n_sample_observed_point"]
        dev = self.device = torch.device(sam6d.device)
        self.meshes = [render.upload(meshio.Mesh(vertices=m.vertices, faces=m.faces), dev) for m in meshes]
        self.icp = pipeline.build_pose_inputs(meshes, objects.model_points_m, dev, icp=True).icp
        mp = torch.from_numpy(np.ascontiguousarray(objects.model_points_m, dtype=np.float32)).to(dev)
        self.icp_radius = mp.norm(dim=2).amax(dim=1).contiguous()                       # as pipeline.icp_refine_out
        mp64 = np.asarray(objects.model_points_m, np.float64)
        centroid = mp64.mean(axis=1)
        self.centroid = torch.from_numpy(centroid.astype(np.float32)).to(dev)
        self.rho = np.linalg.norm(mp64 - centroid[:, None], axis=2).max(axis=1)         # the object's radius about its centroid
        self.gate_radius = torch.from_numpy((self.gate_scale * self.rho).astype(np.float32)).to(dev)
        self.reset()

    def reset(self):
        """drop every track; the next frame runs detection"""
        S = len(self.obj)
        self.R = torch.full((S, 3, 3), float("nan"), device=self.device)
        self.t = torch.full((S, 3), float("nan"), device=self.device)
        self.live = np.zeros(S, bool)
        self.score = np.zeros(S)
        self.frames_tracked = np.zeros(S, np.int64)
        self.track_id = np.full(S, -1, np.int64)
        self._next_id = 0
        self._since_detection = None            # None: no detection since construction or reset()
        self._lost = False

    def start(self, o: int, R, t, score: float = 1.0) -> int:
        """seed a track of object o at pose R (3,3), t (3,) in metres in o's lowest free slot -> its track id.  Raises when o
        has no free slot; with max_instances 1 the new track replaces o's live one, if any."""
        slot = self._free_slot(int(o))
        if slot is None:
            raise ValueError(f"Tracker.start: object {o} already has {self.max_instances} live tracks")
        self._seed(slot, torch.as_tensor(R, dtype=torch.float32, device=self.device).reshape(3, 3),
                   torch.as_tensor(t, dtype=torch.float32, device=self.device).reshape(3), score)
        return int(self.track_id[slot])

    def _free_slot(self, o: int):
        I = self.max_instances
        if I == 1:
            return o
        free = np.flatnonzero(~self.live[o * I:(o + 1) * I])
        return o * I + int(free[0]) if len(free) else None

    def _seed(self, slot: int, R, t, score: float):
        self.R[slot], self.t[slot] = R, t
        self.live[slot], self.score[slot], self.frames_tracked[slot] = True, float(score), 0
        self.track_id[slot], self._next_id = self._next_id, self._next_id + 1

    def _drop(self, slot: int):
        self.live[slot] = False
        self.R[slot], self.t[slot] = float("nan"), float("nan")
        self.track_id[slot] = -1

    def detection_due(self) -> bool:
        return self._since_detection is None or self._lost or self._since_detection >= self.redetect_interval

    def __call__(self, rgb_u8: np.ndarray, depth_raw: np.ndarray, cam_K, depth_scale):
        """one frame: rgb (H,W,3) u8, depth (H,W) raw u16, cam_K (9 values), depth_scale as camera.json holds them ->
        SimpleNamespace(R (S,3,3), t (S,3) metres on the device for the S = O x max_instances slots, NaN rows for free slots;
        state (S) "tracked", "detected" or "absent"; inliers (S) and rms (S) metres of the tracking ICP (-1 and NaN where it did
        not run); track_id (S) int64, -1 for a free slot; obj (S) each slot's object; records, one per live track with
        pem_records' keys plus track and frames_tracked (and track_id when max_instances > 1); detection, detect_objects'
        result when detection ran on this frame, else None)"""
        t0 = time.time()
        S = len(self.obj)
        H, W = depth_raw.shape
        K = np.asarray(cam_K, np.float64).reshape(3, 3)
        state = [ABSENT] * S
        inliers, rms = np.full(S, -1, np.int64), np.full(S, np.nan)
        live = np.flatnonzero(self.live)
        cand = None
        if len(live):
            cand = self._track(live, np.ascontiguousarray(depth_raw, dtype=np.uint16), K, depth_scale, H, W, inliers, rms)
            for s in live:
                if self.live[s]:
                    state[s] = TRACKED
                    self.frames_tracked[s] += 1
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
        return SimpleNamespace(R=self.R.clone(), t=self.t.clone(), state=state, inliers=inliers, rms=rms, track_id=self.track_id.copy(),
                               obj=self.obj.copy(), records=records, detection=detection)

    def _track(self, live, depth_raw, K, depth_scale, H, W, inliers, rms):
        """render, select points and refine every live track; drop the tracks the loss rule, and with max_instances > 1 the
        merge rule, rejects -> the candidate masks"""
        idx = torch.from_numpy(live).to(self.device)
        oidx = torch.from_numpy(self.obj[live]).to(self.device)
        R, t = self.R[idx].contiguous(), self.t[idx].contiguous()
        poses = torch.zeros(len(live), 1, 4, 4, device=self.device)
        poses[:, 0, :3, :3] = R
        poses[:, 0, :3, 3] = t * 1000.0                                                   # the meshes are in mm
        poses[:, 0, 3, 3] = 1.0
        rdepth = render.render([self.meshes[o] for o in self.obj[live]], poses, K, H, W)["depth"][:, 0].contiguous()
        centre = (torch.einsum("lij,lj->li", R, self.centroid[oidx]) + t).contiguous()
        depth_d = torch.from_numpy(depth_raw).to(self.device)
        select = ops.track_points if self.max_instances == 1 else ops.track_points_scene
        pts, _, cand = select(rdepth, depth_d, depth_scale, K, centre, self.gate_radius[oidx].contiguous(), self.margin_px, self.n_points)
        R1, t1, inl, err, _ = ops.icp_refine(R, t, pts, self.icp[0], self.icp[1], oidx.to(torch.int32), self.icp_radius[oidx].contiguous(),
                                             self.track_icp_iters)
        inl, err = inl.cpu().numpy(), err.cpu().numpy()
        self.R[idx], self.t[idx] = R1, t1
        for j, s in enumerate(live):
            inliers[s], rms[s] = inl[j], err[j]
            if inl[j] < self.min_inlier_fraction * self.n_points or err[j] > self.max_rms_m:
                self._drop(s)
        if self.max_instances > 1:
            self._merge()
        return cand

    def _centroids(self, R, t, o):
        """(k,3,3), (k,3) poses of object o -> (k,3) float64 centroids R c_o + t in metres"""
        R, t = np.asarray(R, np.float64).reshape(-1, 3, 3), np.asarray(t, np.float64).reshape(-1, 3)
        return np.einsum("kij,j->ki", R, self.centroid[o].cpu().numpy().astype(np.float64)) + t

    def _merge(self):
        """per object, walking its live tracks by ascending id: drop a track whose centroid lies within assoc_scale x rho of a
        kept (older) track's"""
        R, t = self.R.cpu().numpy(), self.t.cpu().numpy()
        for o in range(len(self.objects.obj_ids)):
            slots = list(np.flatnonzero(self.live & (self.obj == o)))
            slots.sort(key=lambda s: self.track_id[s])
            kept = []
            for s, c in zip(slots, self._centroids(R[slots], t[slots], o)):
                if any(np.linalg.norm(c - k) <= self.assoc_scale * self.rho[o] for k in kept):
                    self._drop(s)
                else:
                    kept.append(c)

    def _start_from(self, det, state):
        """start tracks from detect_objects' result -> {slot: the PEM record that started it}.  With max_instances 1, each
        object with no live track starts from its highest-scoring PEM instance; else see _start_instances"""
        frame, started = det.frame, {}
        if frame is None or frame.out is None or not det.pem:
            return started
        obj, scores = np.asarray(frame.obj), np.asarray(frame.pose_scores)
        if self.max_instances > 1:
            return self._start_instances(det, obj, scores, state)
        for o in range(len(state)):
            rows = np.flatnonzero(obj == o)
            if self.live[o] or not len(rows):
                continue
            best = int(rows[np.argmax(scores[rows])])                                   # the first of equal scores
            self._seed(o, det.R[best], det.t[best], float(scores[best]))
            started[o] = dict(det.pem[best])
            state[o] = DETECTED
        return started

    def _start_instances(self, det, obj, scores, state):
        """per object, its PEM instances by descending score (stable): with no live track the best starts whatever its score;
        every further one needs score >= start_score and a centroid farther than assoc_scale x rho from every live track of
        the object, those started here included; until the object's slots are full"""
        started = {}
        R, t = self.R.cpu().numpy(), self.t.cpu().numpy()
        dR, dt = det.R.cpu().numpy(), det.t.cpu().numpy()
        for o in range(len(self.objects.obj_ids)):
            rows = np.flatnonzero(obj == o)
            if not len(rows):
                continue
            mine = np.flatnonzero(self.live & (self.obj == o))
            live = list(self._centroids(R[mine], t[mine], o))
            for i in rows[np.argsort(-scores[rows], kind="stable")]:
                slot = self._free_slot(o)
                if slot is None:
                    break
                c = self._centroids(dR[i], dt[i], o)[0]
                if live and (scores[i] < self.start_score or any(np.linalg.norm(c - k) <= self.assoc_scale * self.rho[o] for k in live)):
                    continue
                self._seed(slot, det.R[i], det.t[i], float(scores[i]))
                started[slot] = dict(det.pem[i])
                state[slot] = DETECTED
                live.append(c)
        return started

    def _records(self, state, started, cand, live, hw, runtime):
        """one record per live track: a detected track's PEM record, a tracked one's pose with the bbox and RLE of its
        candidate pixels; each with track (the state) and frames_tracked, and track_id when max_instances > 1"""
        S = len(state)
        R, t = self.R.cpu().numpy(), self.t.cpu().numpy() * 1000.0
        rec = [None] * S
        tracked = [s for s in range(S) if state[s] == TRACKED]
        if tracked:
            rows = [int(np.flatnonzero(live == s)[0]) for s in tracked]
            m = cand[torch.tensor(rows, device=cand.device)]
            cum, off = ops.mask_rle(m.float().contiguous())
            counts = pipeline.rle_counts(cum.cpu().numpy(), off.cpu().numpy())
            ys, xs = m.any(dim=2).cpu().numpy(), m.any(dim=1).cpu().numpy()
            for j, s in enumerate(tracked):
                y, x = np.flatnonzero(ys[j]), np.flatnonzero(xs[j])
                bbox = [int(x[0]), int(y[0]), int(x[-1] + 1 - x[0]), int(y[-1] + 1 - y[0])] if len(x) else [0, 0, 0, 0]
                rec[s] = dict(scene_id=0, image_id=0, category_id=int(self.objects.obj_ids[self.obj[s]]), bbox=bbox,
                              score=float(self.score[s]), time=float(runtime),
                              segmentation={"counts": counts[j], "size": [int(hw[0]), int(hw[1])]})
        for s in range(S):
            if state[s] == DETECTED:
                rec[s] = started[s]
            if rec[s] is not None:
                rec[s].update(R=R[s].tolist(), t=t[s].tolist(), track=state[s], frames_tracked=int(self.frames_tracked[s]))
                if self.max_instances > 1:
                    rec[s]["track_id"] = int(self.track_id[s])
        return [r for r in rec if r is not None]
