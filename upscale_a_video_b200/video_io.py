"""Host-side file I/O of the `python -m upscale_a_video_b200` command, with OpenCV: input discovery, frame reading and
output writing (the reference's `utils.py` `get_video_paths` / `read_frame_from_videos` and the saving block of
`inference_upscale_a_video.py:340-361`).

Frames stay uint8 in OpenCV's BGR order until they are on the GPU (`ops.unpack_video_uint8`); writers take RGB uint8
frames `(t, h, w, 3)` and reverse the channels at write time.  OpenCV is imported on first use, so the library itself
does not need it."""
from __future__ import annotations

import os
from typing import List, Optional, Tuple

import numpy as np

IMAGE_EXTENSIONS = (".jpg", ".jpeg", ".png")
VIDEO_EXTENSIONS = (".mp4", ".mov", ".avi")
# an image folder has no frame rate; the reference writes its mp4 with imageio's ffmpeg writer, whose default is 10
DEFAULT_FPS = 10


def _cv2():
    try:
        import cv2
    except ImportError as e:
        raise ImportError("reading and writing video files needs OpenCV (the `cv2` module)") from e
    return cv2


def is_video(path: str) -> bool:
    return path.lower().endswith(VIDEO_EXTENSIONS)


def is_image(path: str) -> bool:
    return path.lower().endswith(IMAGE_EXTENSIONS)


def get_video_paths(input_root: str) -> List[str]:
    """every video file under `input_root`, recursively, sorted (utils.py:28-34)"""
    paths = []
    for root, _, files in os.walk(input_root):
        paths.extend(os.path.join(root, f) for f in files if is_video(f))
    return sorted(paths)


def find_inputs(input_path: str) -> List[str]:
    """inference_upscale_a_video.py:139-150: a video file, an image folder (one clip) or a folder of videos.  A folder is
    classified by its first entry in sorted order (the reference takes the first entry of an unsorted listdir)."""
    if is_video(input_path):
        if not os.path.isfile(input_path):
            raise FileNotFoundError(f"input video {input_path} does not exist")
        return [input_path]
    if os.path.isdir(input_path):
        entries = sorted(os.listdir(input_path))
        if entries and is_image(entries[0]):
            return [input_path]
        if entries and is_video(entries[0]):
            return get_video_paths(input_path)
    raise ValueError(f"Invalid input: '{input_path}' should be a path to a video file, a folder of images or a folder "
                     "containing videos.")


def read_frames(path: str) -> Tuple[np.ndarray, Optional[float], str]:
    """utils.py:9-25 without the float conversion: returns (frames (t, h, w, 3) uint8 BGR, fps, video name).  A video's fps
    is its CAP_PROP_FPS; an image folder (its image files in name order) has fps None."""
    cv2 = _cv2()
    if is_video(path):
        name = os.path.splitext(os.path.basename(path))[0]
        cap = cv2.VideoCapture(path)
        if not cap.isOpened():
            raise RuntimeError(f"OpenCV cannot open the video {path}")
        fps = cap.get(cv2.CAP_PROP_FPS)
        frames = []
        while True:
            ok, frame = cap.read()
            if not ok:
                break
            frames.append(frame)
        cap.release()
        fps = fps if fps > 0 else None
    else:
        name = os.path.basename(os.path.normpath(path))
        fps = None
        frames = []
        for f in sorted(os.listdir(path)):
            if not is_image(f):
                continue
            frame = cv2.imread(os.path.join(path, f), cv2.IMREAD_COLOR)
            if frame is None:
                raise RuntimeError(f"OpenCV cannot read the image {os.path.join(path, f)}")
            frames.append(frame)
    if not frames:
        raise RuntimeError(f"no frames in {path}")
    if any(f.shape != frames[0].shape for f in frames):
        raise ValueError(f"the frames of {path} differ in size")
    return np.stack(frames), fps, name


def read_first_frame(path: str) -> np.ndarray:
    """frame 0 of a clip, (h, w, 3) uint8 BGR, equal to `read_frames(path)[0][0]` without reading the other frames"""
    cv2 = _cv2()
    if is_video(path):
        cap = cv2.VideoCapture(path)
        if not cap.isOpened():
            raise RuntimeError(f"OpenCV cannot open the video {path}")
        ok, frame = cap.read()
        cap.release()
        if not ok:
            raise RuntimeError(f"no frames in {path}")
        return frame
    for f in sorted(os.listdir(path)):
        if is_image(f):
            frame = cv2.imread(os.path.join(path, f), cv2.IMREAD_COLOR)
            if frame is None:
                raise RuntimeError(f"OpenCV cannot read the image {os.path.join(path, f)}")
            return frame
    raise RuntimeError(f"no frames in {path}")


class VideoWriter:
    """mp4 (fourcc mp4v) written chunk by chunk: opened once for frames of (h, w), then `write((t, h, w, 3) uint8 RGB)`
    per chunk; fps None -> DEFAULT_FPS.  A context manager: the file is finalised when the block ends."""

    def __init__(self, path: str, fps: Optional[float], size: Tuple[int, int]):
        cv2 = _cv2()
        self.path, self.size = path, tuple(size)
        h, w = self.size
        self._writer = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"mp4v"), float(fps or DEFAULT_FPS), (w, h))
        if not self._writer.isOpened():
            raise RuntimeError(f"OpenCV cannot write the video {path}")

    def write(self, frames_rgb: np.ndarray) -> None:
        t, h, w, c = frames_rgb.shape
        assert c == 3 and frames_rgb.dtype == np.uint8 and (h, w) == self.size
        for frame in frames_rgb:
            self._writer.write(np.ascontiguousarray(frame[..., ::-1]))

    def close(self) -> None:
        self._writer.release()

    def __enter__(self) -> "VideoWriter":
        return self

    def __exit__(self, *exc) -> None:
        self.close()


def write_video(path: str, frames_rgb: np.ndarray, fps: Optional[float]) -> None:
    """mp4 (fourcc mp4v) of (t, h, w, 3) uint8 RGB frames; fps None -> DEFAULT_FPS"""
    with VideoWriter(path, fps, frames_rgb.shape[1:3]) as writer:
        writer.write(frames_rgb)


def write_frames(folder: str, frames_rgb: np.ndarray, start: int = 0) -> List[str]:
    """one PNG per frame of (t, h, w, 3) uint8 RGB frames, numbered from `start`: folder/0000.png, folder/0001.png, ..."""
    cv2 = _cv2()
    os.makedirs(folder, exist_ok=True)
    paths = []
    for i, frame in enumerate(frames_rgb, start):
        p = os.path.join(folder, f"{i:04d}.png")
        if not cv2.imwrite(p, np.ascontiguousarray(frame[..., ::-1])):
            raise RuntimeError(f"OpenCV cannot write {p}")
        paths.append(p)
    return paths
