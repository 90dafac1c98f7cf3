"""Video write-out (SURVEY.md section 8f-3): drop-ins for utils/video_op.py:167-213 `save_i2vgen_video_safe`,
:263-309 `save_t2vhigen_video_safe` and :216-262 `save_video_local` (InstructVideo) that take the decoded video WHERE IT
IS -- on the GPU.

The reference copies [1,3,f,H,W] fp32 to the host (173 MB at config 2), un-normalises / clamps / scales / transposes /
casts on the CPU, and hands uint8 frames to imageio (libx264).  Here one kernel (vgen_video_to_rgb8) produces the
frames as RGB bytes on the device -- bit-identical to the reference's arithmetic -- they cross PCIe once into pinned
memory (4x fewer bytes), and are piped as rawvideo to an `ffmpeg` process (libx264, yuv420p).  `async_=True` does
the D2H copy on a side stream and the encoding on a worker thread, so the next prompt's sampling overlaps it.

The last-frame anomaly test (:196-202, "Fix known bugs": drop the last frame when > 40 % of its bytes are in
[117, 137]) is evaluated from a per-frame counter the same kernel fills.
Encoders: `ffmpeg` on PATH (same codec / pixel format as the reference), else OpenCV's VideoWriter (mp4v); a single
frame is written as PNG like the reference.  Neither available -> VgenError (frames are never silently discarded).
"""
from __future__ import annotations

import os
import shutil
import subprocess
import threading

import torch

from . import ops
from .lib import VgenError


def frames_to_host(gen_video, mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5), stream=None):
    """gen_video [b,3,f,h,w] (CUDA, any float dtype; batch entry 0 is written, like the reference) ->
    (pinned uint8 [f,h,w,3], pinned int64 [f] band counts, event recorded after the D2H copies)."""
    if not gen_video.is_cuda:
        raise VgenError("vgen_b200.video_io: gen_video must be a CUDA tensor (the reference's .cpu() call is not needed)")
    if gen_video.dim() != 5 or gen_video.shape[1] != 3:
        raise ValueError("gen_video must be [b, 3, f, h, w]")
    v = gen_video[0]
    v = v if (v.dtype == torch.float32 and v.is_contiguous()) else v.float().contiguous()
    cur = torch.cuda.current_stream(v.device)
    side = stream or cur
    if side is not cur:
        side.wait_stream(cur)
    with torch.cuda.stream(side):
        rgb, band = ops.video_to_rgb8(v, mean, std)
        host = torch.empty(rgb.shape, dtype=torch.uint8, pin_memory=True)
        hband = torch.empty(band.shape, dtype=torch.int64, pin_memory=True)
        host.copy_(rgb, non_blocking=True)
        hband.copy_(band, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(side)
        v.record_stream(side)
    return host, hband, ev


def select_frames(host, hband):
    """:196-202 on the kernel's counters: returns the number of leading frames to encode."""
    f = host.shape[0]
    if f > 1 and int(hband[f - 1]) / float(host[f - 1].numel()) > 0.4:
        return f - 1
    return f


def _encode(local_path, frames, save_fps, video=False):
    """frames: uint8 numpy [n,h,w,3] RGB.  One frame is written as a PNG unless `video` asks for the video file anyway."""
    n, h, w, _ = frames.shape
    os.makedirs(os.path.dirname(os.path.abspath(local_path)), exist_ok=True)
    if n == 1 and not video:
        import cv2
        cv2.imwrite(local_path + ".png", frames[0][:, :, ::-1], [int(cv2.IMWRITE_JPEG_QUALITY), 100])
        return local_path + ".png"
    ff = shutil.which("ffmpeg")
    if ff:
        cmd = [ff, "-y", "-loglevel", "quiet", "-f", "rawvideo", "-pix_fmt", "rgb24", "-s", f"{w}x{h}", "-r", str(save_fps),
               "-i", "-", "-vcodec", "libx264", "-crf", "17", "-pix_fmt", "yuv420p", local_path]
        p = subprocess.Popen(cmd, stdin=subprocess.PIPE)
        p.stdin.write(memoryview(frames).cast("B"))
        p.stdin.close()
        if p.wait() != 0:
            raise VgenError(f"ffmpeg exited with {p.returncode} writing {local_path}")
        return local_path
    try:
        import cv2
        wr = cv2.VideoWriter(local_path, cv2.VideoWriter_fourcc(*"mp4v"), float(save_fps), (w, h))
        if not wr.isOpened():
            raise VgenError("cv2.VideoWriter could not open the output")
        for fr in frames:
            wr.write(fr[:, :, ::-1])
        wr.release()
        return local_path
    except ImportError as e:
        raise VgenError("vgen_b200.video_io: neither `ffmpeg` nor OpenCV is available to encode the video") from e


class _Pending:
    def __init__(self, thread, box):
        self._t, self._box = thread, box

    def join(self):
        self._t.join()
        if "error" in self._box:
            raise self._box["error"]
        return self._box.get("path")


_SIDE = {}


@torch.no_grad()
def save_i2vgen_video_safe(local_path, gen_video, captions=None, mean=[0.5, 0.5, 0.5], std=[0.5, 0.5, 0.5], text_size=256,
                           retry=5, save_fps=8, async_=False):
    """utils/video_op.py:167-213 (same signature; gen_video stays on the GPU).  async_=True returns a handle whose
    .join() waits for the file; the device work and the copy run on a side stream."""
    if async_:
        dev = gen_video.device
        side = _SIDE.get(dev) or _SIDE.setdefault(dev, torch.cuda.Stream(dev))
        host, hband, ev = frames_to_host(gen_video, mean, std, stream=side)
        box = {}

        def work():
            try:
                ev.synchronize()
                n = select_frames(host, hband)
                box["path"] = _encode(local_path, host[:n].numpy(), save_fps)
            except Exception as e:  # noqa: BLE001 - re-raised by join()
                box["error"] = e
        th = threading.Thread(target=work, daemon=True)
        th.start()
        return _Pending(th, box)
    host, hband, ev = frames_to_host(gen_video, mean, std)
    ev.synchronize()
    n = select_frames(host, hband)
    exc = None
    for _ in range(max(1, retry)):
        try:
            return _encode(local_path, host[:n].numpy(), save_fps)
        except Exception as e:  # noqa: BLE001 - the reference retries the encoder the same way (:193-210)
            exc = e
    raise exc


save_t2vhigen_video_safe = save_i2vgen_video_safe   # identical body in the reference (:263-309)


@torch.no_grad()
def save_video_local(local_path, gen_video, mean=[0.5, 0.5, 0.5], std=[0.5, 0.5, 0.5], retry=5):
    """utils/video_op.py:216-262 (InstructVideo's writer, same signature): the frames of batch entry 0 with the same
    arithmetic as save_i2vgen_video_safe but no last-frame drop, written to local_path as an 8 fps mp4 (libx264, crf 17,
    yuv420p) even for a single frame.  Returns the f frames as uint8 numpy [h, w, 3] RGB, like the reference.
    gen_video is not modified (the reference un-normalises it in place).  The InstructVideo entrance passes a host tensor
    (gen_videos.cpu(), inference_instructvideo_entrance.py:264); it is copied to the current CUDA device, where the
    frames are made -- passing the CUDA tensor saves the round trip."""
    if not gen_video.is_cuda:
        gen_video = gen_video.to(torch.device("cuda", torch.cuda.current_device()))
    host, _band, ev = frames_to_host(gen_video, mean, std)
    ev.synchronize()
    frames = host.numpy().copy()
    exc = None
    for _ in range(max(1, retry)):
        try:
            _encode(local_path, frames, 8, video=True)
            return list(frames)
        except Exception as e:  # noqa: BLE001 - retried like the reference (:241-257)
            exc = e
    raise exc
