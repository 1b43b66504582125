"""Python mirror of the reference's detector class surface, over the C ABI.

Mirrors ``class RetinaFace`` (retinaface/RetinaFace.h:63-70): same constructor arguments
(model directory, network name "net3", nms threshold 0.4), ``detect(img, threshold, scales)``
and ``detectBatchImages(imgs, threshold)``.  The reference's methods return ``void`` and drop
their results (RetinaFace.cpp:665,726,747); here they return the ``FaceDetectInfo`` list that the
reference computes and discards.  The C++ twin of this file is ``retinaface_b200/host/RetinaFace.h``.
"""
from __future__ import annotations

import os
from dataclasses import dataclass
from typing import List, Sequence

import numpy as np

from .capi import ANY_ORIENTATION, CROP_FORMATS, RF_PREC_FP16, Engine, crop_shape


@dataclass
class FaceDetectInfo:  # RetinaFace.h:37-42
    score: float
    rect: tuple   # anchor_box x1,y1,x2,y2
    pts_x: tuple  # FacePts.x[5]
    pts_y: tuple  # FacePts.y[5]

    @staticmethod
    def from_row(r: np.ndarray) -> "FaceDetectInfo":
        return FaceDetectInfo(float(r[0]), tuple(map(float, r[1:5])), tuple(map(float, r[5:10])), tuple(map(float, r[10:15])))


def angle_sweep(step: float) -> list:
    """The rotated views of ``detectAnyAngle`` and ``detectAnyAngleFrames``: (angle, shrink 1) for the angles 0, step, 2 step ... below
    360 degrees.  A step that is not positive, or one that makes more than RF_MAX_VIEWS = 16 views, is a ValueError."""
    if not step > 0:
        raise ValueError(f"step {step}: must be positive")
    angles = [0.0]
    while len(angles) <= 16 and len(angles) * float(step) < 360.0:
        angles.append(len(angles) * float(step))
    if len(angles) > 16:
        raise ValueError(f"step {step} makes more than RF_MAX_VIEWS = 16 views")
    return [(a, 1.0) for a in angles]


class RetinaFace:
    MODEL_FILE = "mnet-deconv-0517.caffemodel"  # the file the reference always loads, RetinaFace.cpp:276

    def __init__(self, model: str, network: str = "net3", nms: float = 0.4, *, net_w: int = 448, net_h: int = 448,
                 max_batch: int = 8, precision: int = RF_PREC_FP16, device: int = 0, max_faces: int = 256,
                 model_file: str = None, max_image=(3072, 4096)):
        if network != "net3":
            # RetinaFace.cpp:211-242 lists other names, but only the fmc==3 "net3" anchors are configured (:245-271)
            raise ValueError(f"network setting error {network}: only 'net3' is configured")
        self.nms_threshold = nms
        path = os.path.join(model, model_file or self.MODEL_FILE)
        self.engine = Engine(path, net_h, net_w, precision=precision, max_batch=max_batch, max_faces=max_faces,
                             device=device, max_image=max_image)

    def detect(self, img: np.ndarray, threshold: float = 0.5, scales: float = 1.0) -> List[FaceDetectInfo]:
        if img is None or img.size == 0:  # RetinaFace.cpp:578-580
            return []
        return self.detectBatchImages([img], threshold)[0]

    def detectBatchImages(self, imgs: Sequence[np.ndarray], threshold: float = 0.5) -> List[List[FaceDetectInfo]]:
        rows = self.engine.detect_batch(list(imgs), threshold, self.nms_threshold)
        return [[FaceDetectInfo.from_row(r) for r in per] for per in rows]

    def detectAndAlign(self, imgs: Sequence[np.ndarray], threshold: float = 0.5, **align) -> List[List[tuple]]:
        """Face alignment on the GPU (f5): per image, a list of ``(FaceDetectInfo, crop)`` -- the face in ORIGINAL IMAGE pixels and
        its crop warped from the original image onto a landmark template (``Engine.detect_align``'s keyword arguments: crop,
        template, fmt, max_faces, mean, std; by default 112x112 u8 BGR on the ArcFace template).  With ``max_faces`` only the
        best-scoring faces of each image are returned."""
        faces, crops = self.engine.detect_align(list(imgs), threshold, self.nms_threshold, **align)
        return [[(FaceDetectInfo.from_row(r), c) for r, c in zip(f, cs)] for f, cs in zip(faces, crops)]

    def detectFrames(self, frames: Sequence, threshold: float = 0.5, layout: str = "nv12", matrix: str = "bt601", align: dict = None):
        """f6 video frames: 8-bit YUV 4:2:0 host frames (OpenCV's single-buffer ``(h * 3 / 2, w)`` u8 arrays in ``layout`` nv12 |
        nv21 | i420 | yv12, or plane tuples; ``matrix`` bt601 (== cv2.COLOR_YUV2BGR_*) | bt709), converted to BGR inside the
        letter-box on the GPU.  Per frame, the faces in FRAME pixels; with ``align`` (``Engine.detect_align``'s keywords), a list
        of ``(FaceDetectInfo, crop)`` as ``detectAndAlign`` returns."""
        out = self.engine.detect_yuv(list(frames), threshold, self.nms_threshold, layout=layout, matrix=matrix, align=align)
        if align is None:
            return [[FaceDetectInfo.from_row(r) for r in per] for per in out]
        faces, crops = out[0], out[1]
        return [[(FaceDetectInfo.from_row(r), c) for r, c in zip(f, cs)] for f, cs in zip(faces, crops)]

    def detectTiled(self, imgs: Sequence[np.ndarray], threshold: float = 0.5, scales: Sequence[float] = None, flip: bool = False,
                    overlap: int = 0, align: dict = None, orientations: Sequence[int] = None) -> List[list]:
        """f7 small faces in large images: each image is resized to a pyramid of levels, every level cut into overlapping
        network-sized tiles, the tiles detected as ordinary batches and the faces merged across tiles and levels on the GPU
        (rf_detect_tiled).  Faces in ORIGINAL IMAGE pixels.  ``scales``: the levels (a scale may exceed 1; 0 is the letter-box of
        ``detectBatchImages``), each also run mirrored with ``flip``; None: the default pyramid 1, 1/2, 1/4, ... down to the
        letter-box; ``flip`` needs explicit ``scales`` (ValueError otherwise).  ``overlap``: pixels neighbouring tiles share (0: 64).
        With ``align`` (``Engine.detect_align``'s keywords), per image a list of ``(FaceDetectInfo, crop)`` as ``detectAndAlign``
        returns, the crops cut from the original image (rf_detect_tiled_align).  ``orientations`` (f21): image i is shown in EXIF
        orientation ``orientations[i]`` and tiled as displayed, faces and crops in DISPLAYED image pixels (rf_detect_tiled_oriented);
        None: the images as stored."""
        if flip and scales is None:
            raise ValueError("detectTiled: flip mirrors the given scales; the default pyramid has no mirrored levels -- pass scales")
        levels = None if scales is None else [(float(s), f) for s in scales for f in ((False, True) if flip else (False,))]
        if orientations is None:
            out = self.engine.detect_tiled(list(imgs), threshold, self.nms_threshold, levels=levels, overlap=overlap, align=align)
        else:
            out = self.engine.detect_tiled_oriented(list(imgs), list(orientations), threshold, self.nms_threshold, levels=levels,
                                                    overlap=overlap, align=align)
        if align is None:
            return [[FaceDetectInfo.from_row(r) for r in per] for per in out[0]]
        return [[(FaceDetectInfo.from_row(r), c) for r, c in zip(f, cs)] for f, cs in zip(out[0], out[2])]

    def detectInImage(self, img: np.ndarray, threshold: float = 0.5, scales: Sequence[float] = (1.0,), flip: bool = False
                      ) -> List[FaceDetectInfo]:
        """SURVEY.md 8f-2: what the reference leaves commented out / unused (RetinaFace.cpp:730-746, the `scales` argument of
        RetinaFace.h:70): faces in ORIGINAL IMAGE pixels (x * scale), optionally with multi-scale + horizontal-flip test-time
        augmentation.  ``scales``: fractions (0, 1] of the network input the image is fitted into; with ``flip`` every scale
        is also run mirrored.  All views form one batch; the merge NMS across views runs on the GPU (rf_detect_views)."""
        if img is None or img.size == 0:
            return []
        views = [(float(s), f) for s in scales for f in ((False, True) if flip else (False,))]
        faces, _, _ = self.engine.detect_views(img, views, threshold, self.nms_threshold)
        return [FaceDetectInfo.from_row(r) for r in faces]

    def detectOriented(self, imgs: Sequence[np.ndarray], orientations: Sequence[int], threshold: float = 0.5, align: dict = None) -> List[list]:
        """f9 rotated and mirrored images: image i as stored, shown in EXIF orientation ``orientations[i]`` (1..8, what cv::imread
        applies; ``capi.exif_orientation`` reads it from JPEG bytes).  Per image, the faces in DISPLAYED image pixels, found and
        cropped without a rotated copy (rf_detect_oriented_batch); with ``align`` (``Engine.detect_align``'s keywords), a list of
        ``(FaceDetectInfo, crop)`` cut from the displayed image."""
        out = self.engine.detect_oriented(list(imgs), list(orientations), threshold, self.nms_threshold, align=align)
        if align is None:
            return [[FaceDetectInfo.from_row(r) for r in per] for per in out]
        return [[(FaceDetectInfo.from_row(r), c) for r, c in zip(f, cs)] for f, cs in zip(out[0], out[1])]

    def detectAnyOrientation(self, img: np.ndarray, threshold: float = 0.5) -> List[FaceDetectInfo]:
        """f9 unknown orientation: the image in its four rotations (EXIF 1, 6, 3, 8) as one batch, merged on the GPU
        (rf_detect_views_oriented).  Faces in STORED image pixels, landmarks on the subject's sides, so an aligned crop of a
        sideways face comes out upright."""
        if img is None or img.size == 0:
            return []
        faces, _, _ = self.engine.detect_views_oriented(img, [(1.0, o) for o in ANY_ORIENTATION], threshold, self.nms_threshold)
        return [FaceDetectInfo.from_row(r) for r in faces]

    def detectAnyAngle(self, img: np.ndarray, threshold: float = 0.5, step: float = 30.0, align: dict = None) -> list:
        """f23 faces at any in-plane angle: the image rotated counter-clockwise by 0, step, 2 step ... below 360 degrees, each view fitted
        into the network input (rf_detect_views_rotated; quarter turns take detectAnyOrientation's views), merged on the GPU.  Faces in
        image pixels, axis-aligned boxes, landmarks carrying each face's roll.  With ``align`` (``Engine.detect_align``'s keywords), a list
        of ``(FaceDetectInfo, crop)``, the crops upright.  More than 16 views (RF_MAX_VIEWS) is a ValueError."""
        views = angle_sweep(step)
        if img is None or img.size == 0:
            return []
        out = self.engine.detect_views_rotated(img, views, threshold, self.nms_threshold, align=align)
        if align is None:
            return [FaceDetectInfo.from_row(r) for r in out[0]]
        return [(FaceDetectInfo.from_row(r), c) for r, c in zip(out[0], out[4])]

    def detectAnyAngleFrames(self, device_frames: Sequence, threshold: float = 0.5, step: float = 30.0, layout: str = "nv12",
                             matrix: str = "bt601") -> List[List[FaceDetectInfo]]:
        """f24 faces at any in-plane angle in video: ``detectAnyAngle``'s sweep on device 4:2:0 frames (torch CUDA tensors in
        ``Engine.detect_yuv_device``'s forms, at most max_batch), all frames in one asynchronous call
        (rf_detect_yuv_views_rotated_device).  Per frame, the faces in FRAME pixels.  More than 16 views is a ValueError."""
        views = angle_sweep(step)
        frames = list(device_frames)
        if not frames:
            return []
        d, c, _, _ = self.engine.detect_yuv_views_rotated_device(frames, views, threshold, self.nms_threshold, layout=layout, matrix=matrix)
        faces, _ = self.engine.read_dets(d, c, len(frames))
        return [[FaceDetectInfo.from_row(r) for r in per] for per in faces]

    def setVideoOrientation(self, video: int, orientation: int):
        """f20 oriented video (rf_tracker_set_orientation): ``video`` (-1: every video) is shown in EXIF orientation 1..8 -- portrait
        phone video stored as landscape surfaces -- and ``trackFrames`` / ``redactFrames`` read and write its frames as displayed, with
        tracks in displayed pixels.  Applied when this detector's tracker is created, or at once when it exists; before the video's
        first tracked frame since creation or a reset."""
        trk = getattr(self, "_tracker", None)
        if trk is not None:
            trk.set_orientation(video, orientation)
        self._orientations = getattr(self, "_orientations", []) + [(int(video), int(orientation))]

    def _new_tracker(self, **kw):
        """Engine.tracker with this detector's video orientations applied."""
        trk = self.engine.tracker(**kw)
        try:
            for v, o in getattr(self, "_orientations", []):
                trk.set_orientation(v, o)
        except Exception:
            trk.close()
            raise
        return trk

    def _interval_calls(self, videos: Sequence[int], detect_every: int):
        """f16: frame i of video v is a detect frame when v's frame number (counted over every call since the tracker's creation or
        the video's reset) is divisible by detect_every.  Returns [(detect?, frame indices)] in issue order: each video's frames split
        into runs of one kind, the p-th runs of every video after the (p - 1)-th, detect before follow -- so each video's frames keep
        their order and a call of one kind stays one call."""
        nums = self.__dict__.setdefault("_frame_no", {})
        runs, seg = {}, {}
        for i, v in enumerate(videos):
            v = int(v)
            det = nums.get(v, 0) % detect_every == 0
            nums[v] = nums.get(v, 0) + 1
            p, last = seg.get(v, (-1, None))
            if det != last:
                p += 1
            seg[v] = (p, det)
            runs.setdefault((p, not det), []).append(i)
        return [(not follow, idx) for (_, follow), idx in sorted(runs.items())]

    def _interval_tracker(self, detect_every: int, best=None, lookback=0, tiling=None, live=None, any_angle=None):
        if int(detect_every) < 1:
            raise ValueError(f"detect_every {detect_every}, must be >= 1")
        if any_angle is not None and tiling:
            raise ValueError("any_angle and tiling are exclusive: a rotated view is not tiled")
        if live is not None and best is None:
            raise ValueError("live shots need best shots: pass best as well")
        trk = getattr(self, "_tracker", None)
        if live is not None and trk is not None and not trk.best_live_on:
            raise ValueError("live: this detector's tracker was created without live shots (the first call decides)")
        if detect_every > 1 and best is not None and trk is not None and not trk.best_follow_on:
            raise ValueError("detect_every > 1 with best shots needs a following best-shot tracker: this detector's tracker was created "
                             "without one (the first call decides the tracker)")
        if detect_every > 1 and lookback and trk is not None and not trk.lookback_follow_on:
            raise ValueError("detect_every > 1 with lookback needs a following look-back tracker: this detector's tracker was created "
                             "without one (the first call decides the tracker)")
        if detect_every > 1 and best is None and not lookback and trk is not None and not trk.follow_on:
            raise ValueError("detect_every > 1 needs a follow tracker: this detector's tracker was created without one")
        if tiling and trk is not None and not trk.tiling_on:
            raise ValueError("tiling: this detector's tracker was created without tiling (the first call decides)")
        if any_angle is not None and trk is not None and not trk.views_on:
            raise ValueError("any_angle: this detector's tracker was created without rotated views (the first call decides)")

    @staticmethod
    def _views(any_angle):
        """The tracker's rotated views of ``any_angle`` (None: none), ``detectAnyAngleFrames``' sweep."""
        return None if any_angle is None else angle_sweep(any_angle)

    def trackFrames(self, frames: Sequence, videos: Sequence[int], threshold: float = 0.5, layout: str = "nv12", matrix: str = "bt601",
                    align: dict = None, max_videos: int = 64, best: dict = None, motion=False, detect_every: int = 1, tiling=None,
                    live=None, any_angle=None):
        """f10 tracking: device 4:2:0 frames (torch CUDA tensors in ``Engine.detect_yuv_device``'s forms), frame i of video
        ``videos[i]``, detected and associated with the tracks of earlier frames on the GPU (rf_detect_yuv_track_device).  Per frame, a
        list of ``(id, state, FaceDetectInfo)`` over every live track (``capi.TRACK_*`` states; the face is the last matched one, in
        FRAME pixels), and per frame a list of ``(id, crop)``: with ``align`` (``Engine.detect_align``'s keywords), one crop per track
        confirmed on that frame -- a new identity -- as a torch CUDA tensor.  The tracker is created on the first call with
        ``max_videos`` sequences; ``resetTracks`` restarts them.

        f11 best shots: with ``best`` (``capi.best_config``'s keywords: crop, template, fmt, mean, std, min_quality, sharp_half) the
        tracker is a best-shot tracker (rf_detect_yuv_track_best_device; ``align`` must then be None) and the second list holds, per
        frame, a ``(shot, crop)`` for every track that ended on that frame: ``shot`` a ``capi.BEST_DTYPE`` record (the quality terms
        and the record of the track's best frame), ``crop`` that frame's crop as a torch CUDA tensor.  ``finishVideo`` emits the
        shots of the tracks still live.

        f13 camera motion: with ``motion`` (True, or ``capi.motion_config``'s keywords: search, min_inliers) the tracker estimates
        each frame's global motion from the previous frame of the same video and moves the tracks with it, so that a panning or
        shaking camera keeps the ids; ``Tracker.motion`` (``self._tracker``) reads the estimates.  The first call decides which kind
        of tracker this detector keeps.

        f16 detection interval: with ``detect_every=k`` > 1 the tracker is a follow tracker; each video's frames whose number is
        divisible by k are detected, the others followed by template search without the detector (rf_track_follow_device).  A call
        mixing both kinds is split into detect and follow calls; each video's frames keep their order.  Follow frames have no crops.

        f19 small faces: with ``tiling`` (True, or ``Tracker.set_tiling``'s keywords: levels, overlap) every detect call of the tracker
        detects through the tiles of ``detectTiled`` (rf_tracker_set_tiling), so faces far below the letter-box's smallest anchor in
        4K frames are tracked too.  The first call decides; asking for it on a tracker created without it raises ValueError.

        f22 live cameras: with ``best`` and ``live`` (True, or ``Tracker.set_best_live``'s keywords: first_quality, improve, min_gap)
        the second list also holds the LIVE shots (reason ``capi.BEST_LIVE``) of tracks that are still live: a first good shot, then
        markedly better ones.  With ``best`` and ``detect_every=k`` > 1 the tracker is a following best-shot tracker: detect frames go
        through rf_detect_yuv_track_best_device, follow frames through rf_track_follow_best_device, whose shots (the EXIT shots of the
        tracks removed there) are returned as well.

        f25 tilted cameras: with ``any_angle=step`` every detect call of the tracker detects through ``detectAnyAngleFrames``' sweep of
        rotated views (rf_tracker_set_views), so the faces of a tilted body-worn or overhead camera are tracked, with any of the above
        but ``tiling`` (ValueError).  The first call decides; asking for it on a tracker created without it raises ValueError."""
        if best is not None and align is not None:
            raise ValueError("best shots and new-identity crops are exclusive: pass best or align, not both")
        self._interval_tracker(detect_every, best=best, tiling=tiling, live=live, any_angle=any_angle)
        if getattr(self, "_tracker", None) is None:
            following = detect_every > 1
            self._tracker = self._new_tracker(max_videos=max_videos, best=best, motion=motion, follow=following and best is None, tiling=tiling,
                                              best_live=live, best_follow=following and best is not None, views=self._views(any_angle))
        if self._tracker.best_follow_on and best is not None:
            tracks, shots = [None] * len(frames), [None] * len(frames)
            for det, idx in self._interval_calls(videos, detect_every):
                fr, vi = [frames[i] for i in idx], [videos[i] for i in idx]
                t, c = self._best_call(fr, vi, threshold, layout, matrix, det)
                for j, i in enumerate(idx):
                    tracks[i], shots[i] = t[j], c[j]
            return tracks, shots
        if self._tracker.follow_on:
            tracks, new = [None] * len(frames), [[] for _ in frames]
            for det, idx in self._interval_calls(videos, detect_every):
                fr, vi = [frames[i] for i in idx], [videos[i] for i in idx]
                if det:
                    t, c = self._track_call(fr, vi, threshold, layout, matrix, align)
                else:
                    tp, tc = self._tracker.follow_device(fr, vi, layout=layout)
                    t = self._lists(self._tracker.read(tp, tc, len(idx)))
                    c = [[] for _ in idx]
                for j, i in enumerate(idx):
                    tracks[i], new[i] = t[j], c[j]
            return tracks, new
        if best is not None:
            return self._best_call(frames, videos, threshold, layout, matrix, True)
        return self._track_call(frames, videos, threshold, layout, matrix, align)

    def _best_call(self, frames, videos, threshold, layout, matrix, detect: bool):
        """One best-shot call -- a detect call, or (f22) a follow call of a following best-shot tracker: the lists and the
        (shot, crop) pairs of each frame."""
        n = len(frames)
        crops = self._best_crops(n)
        if detect:
            bp, bc, tp, tc, _, _, _ = self._tracker.detect_yuv_best_device(list(frames), list(videos), threshold, self.nms_threshold,
                                                                          crops.data_ptr(), layout=layout, matrix=matrix)
        else:
            bp, bc, tp, tc = self._tracker.follow_best_device(list(frames), list(videos), crops.data_ptr(), layout=layout)
        tracks = self._lists(self._tracker.read(tp, tc, n))
        shots = self._tracker.read_best(bp, bc, n)
        return tracks, [[(s, crops[i, k]) for k, s in enumerate(per)] for i, per in enumerate(shots)]

    @staticmethod
    def _lists(recs):
        """(id, state, FaceDetectInfo) rows of each frame's TRACK_DTYPE records."""
        return [[(int(r["id"]), int(r["state"]), FaceDetectInfo.from_row(r["face"])) for r in per] for per in recs]

    @staticmethod
    def _crops(n: int, per: int, fmt: str, crop):
        """An uninitialised (n, per, *crop_shape) torch CUDA tensor for crops in `fmt`."""
        import torch
        shape, dt = crop_shape(fmt, crop)
        return torch.empty((n, per) + shape, dtype={np.uint8: torch.uint8, np.float32: torch.float32, np.float16: torch.float16}[dt],
                           device="cuda")

    def _track_call(self, frames, videos, threshold, layout, matrix, align):
        n = len(frames)
        crops = None
        if align is not None:
            crops = self._crops(n, align.get("max_faces") or self.engine.max_faces, align.get("fmt", "bgr_u8"), align.get("crop", (112, 112)))
        tp, tc, _, _, _ = self._tracker.detect_yuv_device(list(frames), list(videos), threshold, self.nms_threshold, layout=layout, matrix=matrix,
                                                          align=align, dev_crops_ptr=crops.data_ptr() if crops is not None else None)
        recs = self._tracker.read(tp, tc, n)
        tracks = self._lists(recs)
        new = [[(int(r["id"]), crops[i, r["crop_slot"]]) for r in per if r["crop_slot"] >= 0] if crops is not None else []
               for i, per in enumerate(recs)]
        return tracks, new

    def redactFrames(self, frames: Sequence, videos: Sequence[int] = None, threshold: float = 0.5, blocks: int = 0, margin: float = 0.0,
                     layout: str = "nv12", matrix: str = "bt601", max_videos: int = 64, motion=False, style: str = "mosaic",
                     shape: str = "rect", detail: int = 0, lookback: int = 0, out: Sequence = None, detect_every: int = 1,
                     lookback_search=False, tiling=None, any_angle=None):
        """f12 redaction: detect on device 4:2:0 frames (torch CUDA tensors in ``Engine.detect_yuv_device``'s forms) and mosaic every
        detected face IN PLACE (rf_detect_yuv_redact_device), ``blocks`` cells across a region's longer side (0: 8; 1: a flat patch),
        each side grown by ``margin`` of the box (0: 0.25).  With ``videos`` (frame i of video ``videos[i]``) the frames are also
        tracked, on this detector's plain tracker (created as ``trackFrames`` creates it), and the predicted box of every face the
        tracker still follows while the detector misses it is redacted too.  Asynchronous: the frames are complete in stream order on
        ``engine.last_stream_ptr()``.  ``motion`` as ``trackFrames``: the lost faces' predicted boxes then follow the camera.  The first
        call decides the tracker.  f14: ``style="blur"`` blurs each region instead (``detail`` 0: 4; 1..64, a larger detail a smaller
        radius; ``blocks`` must then stay 0), and ``shape="ellipse"`` redacts the ellipse inscribed in each region.
        f15: ``lookback=L`` (with ``videos``) makes the tracker a look-back tracker: each frame is kept on the GPU and frame num - L of
        its video, also covered where the faces first detected in the next L frames already were, is written into ``out[i]`` (None:
        the input frame itself, in place).  Returns the emitted frame numbers (-1: nothing emitted yet); ``drainVideo`` emits the rest.
        f16: ``detect_every=k`` (with ``videos``) detects each video's frames whose number is divisible by k and follows the faces on
        the others (rf_track_follow_redact_device), redacting every followed face and every LOST track, as ``trackFrames`` splits.
        f17: ``lookback_search`` (True or ``Tracker.set_lookback_search`` keywords, with ``lookback``) follows every new face back
        through the buffered frames by template search and covers its path as well; the first call decides, and asking for it on a
        tracker created without it raises ValueError.
        f18: ``lookback=L`` with ``detect_every=k`` > 1 makes a following look-back tracker: the frames are split as f16 splits them,
        key frames go through the look-back call and the others through rf_track_follow_redact_lookback_device, and every frame is
        emitted L frames late; with L >= k - 1 a face first detected on a key frame is also covered on the follow frames before it.
        Returns every frame's emitted number in input order.  The first call decides the tracker.
        f19: ``tiling`` (with ``videos``) as ``trackFrames``: every detect call detects through tiles, with any of the above.
        f25: ``any_angle=step`` (with ``videos``) as ``trackFrames``: every detect call detects through rotated views, with any of the
        above but ``tiling``."""
        kw = dict(layout=layout, matrix=matrix, blocks=blocks, margin=margin, style=style, shape=shape, detail=detail)
        if lookback_search and not lookback:
            raise ValueError("lookback_search needs lookback: the search runs through the look-back buffer")
        self._interval_tracker(detect_every, lookback=lookback, tiling=tiling, any_angle=any_angle)
        if videos is None:
            if tiling:
                raise ValueError("tiling needs videos: it is an option of the tracker")
            if any_angle is not None:
                raise ValueError("any_angle needs videos: it is an option of the tracker")
            if lookback:
                raise ValueError("lookback needs videos: the buffered frames belong to a video")
            if detect_every > 1:
                raise ValueError("detect_every needs videos: the frame numbers belong to a video")
            self.engine.detect_yuv_redact_device(list(frames), threshold, self.nms_threshold, **kw)
            return
        interval = detect_every > 1
        if getattr(self, "_tracker", None) is None:
            self._tracker = self._new_tracker(max_videos=max_videos, motion=motion, lookback=lookback or None,
                                                follow=interval and not lookback, lookback_search=lookback_search or None,
                                                lookback_follow=(interval and lookback) or None, tiling=tiling,
                                                views=self._views(any_angle))
        elif lookback_search and not self._tracker.lookback_search_on:
            raise ValueError("lookback_search: this detector's tracker was created without the look-back search (the first call decides)")
        if lookback and self._tracker.lookback_follow_on:
            outs, fkw = list(frames if out is None else out), {k: v for k, v in kw.items() if k != "matrix"}
            nums = np.full(len(frames), -1, np.int32)
            for det, idx in self._interval_calls(videos, detect_every):
                fr, vi, oo = [frames[i] for i in idx], [videos[i] for i in idx], [outs[i] for i in idx]
                if det:
                    got = self._tracker.detect_yuv_redact_lookback_device(fr, vi, oo, threshold, self.nms_threshold, **kw)[0]
                else:
                    got = self._tracker.follow_redact_lookback_device(fr, vi, oo, **fkw)[0]
                nums[idx] = got
            return nums
        if lookback:
            return self._tracker.detect_yuv_redact_lookback_device(list(frames), list(videos), list(frames if out is None else out), threshold,
                                                                   self.nms_threshold, **kw)[0]
        if self._tracker.follow_on:
            fkw = {k: v for k, v in kw.items() if k != "matrix"}
            for det, idx in self._interval_calls(videos, detect_every):
                fr, vi = [frames[i] for i in idx], [videos[i] for i in idx]
                if det:
                    self._tracker.detect_yuv_redact_device(fr, vi, threshold, self.nms_threshold, **kw)
                else:
                    self._tracker.follow_redact_device(fr, vi, **fkw)
            return
        self._tracker.detect_yuv_redact_device(list(frames), list(videos), threshold, self.nms_threshold, **kw)

    def drainVideo(self, video: int, out: Sequence, layout: str = "nv12", blocks: int = 0, margin: float = 0.0, style: str = "mosaic",
                   shape: str = "rect", detail: int = 0):
        """f15: end ``video`` on a look-back tracker (rf_tracker_drain): its buffered frames (at most L, in frame order) go, redacted,
        into ``out[0..)``; then the video restarts.  Returns their frame numbers."""
        if getattr(self, "_tracker", None) is None or not self._tracker.lookback:
            raise ValueError("drainVideo needs a look-back tracker: call redactFrames(..., lookback=L) first")
        nums = self._tracker.drain(video, list(out), layout=layout, blocks=blocks, margin=margin, style=style, shape=shape, detail=detail)
        getattr(self, "_frame_no", {}).pop(video, None)      # the drain restarts the video's numbering: key frames stay aligned
        return nums

    def _best_crops(self, n: int):
        b = self._tracker.best
        fmt = next(k for k, v in CROP_FORMATS.items() if v[0] == b.align.format)
        return self._crops(n, self._tracker.max_tracks, fmt, (b.align.crop_w, b.align.crop_h))

    def finishVideo(self, video: int) -> list:
        """f11: end ``video`` on a best-shot tracker (rf_tracker_finish): a ``(shot, crop)`` for every live track that was ever
        confirmed, in id order, then the video restarts (ids from 1)."""
        if getattr(self, "_tracker", None) is None or self._tracker.best is None:
            raise ValueError("finishVideo needs a best-shot tracker: call trackFrames(..., best=...) first")
        crops = self._best_crops(1)[0]
        bp, bc = self._tracker.finish(video, crops.data_ptr())
        self.__dict__.get("_frame_no", {}).pop(int(video), None)      # the video restarts: its next frame is a detect frame
        shots = self._tracker.read_best(bp, bc, 1)[0]
        return [(s, crops[k]) for k, s in enumerate(shots)]

    def resetTracks(self, video: int = -1):
        """Restart one video's tracks (ids from 1), or every video's with -1."""
        if getattr(self, "_tracker", None) is not None:
            self._tracker.reset(video)
        nums = getattr(self, "_frame_no", {})
        for v in (list(nums) if video < 0 else [video]):
            nums.pop(v, None)

    @staticmethod
    def draw(img: np.ndarray, faces: Sequence[FaceDetectInfo]) -> np.ndarray:
        """The reference's commented-out visualisation (RetinaFace.cpp:730-741): red box outline of thickness 2, green
        landmark dots, on a copy (:744: `clone()`), for faces in image coordinates.  Plain numpy (no OpenCV needed)."""
        out = np.array(img, dtype=np.uint8, copy=True)
        hh, ww = out.shape[:2]

        def fill(x0, y0, x1, y1, colour):
            x0, y0, x1, y1 = max(x0, 0), max(y0, 0), min(x1, ww), min(y1, hh)
            if x1 > x0 and y1 > y0:
                out[y0:y1, x0:x1] = colour
        for f in faces:
            x1, y1, x2, y2 = (int(round(v)) for v in f.rect)
            for (a, b, c, d) in ((x1 - 1, y1 - 1, x2 + 1, y1 + 1), (x1 - 1, y2 - 1, x2 + 1, y2 + 1),
                                 (x1 - 1, y1 - 1, x1 + 1, y2 + 1), (x2 - 1, y1 - 1, x2 + 1, y2 + 1)):
                fill(a, b, c, d, (0, 0, 255))
            for px, py in zip(f.pts_x, f.pts_y):
                cx, cy = int(round(px)), int(round(py))
                fill(cx - 1, cy - 1, cx + 2, cy + 2, (0, 255, 0))
        return out

    @staticmethod
    def map_back_scale(img_w: int, img_h: int, net_w: int, net_h: int) -> float:
        """scale of RetinaFace.cpp:587-591: multiply coordinates by it to return to image pixels (:732-738)."""
        return max(img_w / net_w, img_h / net_h, 1.0)
