"""Input side of the rasterizer path (SURVEY section 8, "next" row f-4): the on-disk format and the per-image dispatcher.

`load_transforms` restates what the reference's dataparser does to a nerfstudio `transforms.json` with this fork's
extensions (nerfstudio/data/dataparsers/nerfstudio_dataparser.py:91-352): frames sorted by file name, global or
per-frame intrinsics, top-level `exposure_time` / `rolling_shutter_time` (seconds, :331-332), per-frame
`camera_linear_velocity` + `camera_angular_velocity` (camera frame, OpenGL axes; :190-198, linear part multiplied by
the pose scale factor, :334-336), "up" orientation + "poses" centring (cameras/camera_utils.py:520-628), auto scale to
the unit box (:268-274), train/eval split (data/utils/dataparsers_utils.py:23-43) and output-resolution rescale (:353).
Pinned against the reference parser itself: tests/golden/make_golden_data.py runs it on fabricated datasets and
tests/test_data_cpu.py compares.  `load_ply_points` reads the seed cloud (`sparse_pc.ply`) into the same frame.

`load_image_u8` / `composite_u8` read and composite a training image like the reference's dataset and model do
(data/datasets/base_dataset.py:61-110, models/splatfacto.py:900-923).

`to_gsplat_camera` is the camera block of Splatfacto.get_outputs (nerfstudio/models/splatfacto.py:733-747,799-800):
OpenGL camera-to-world -> gsplat world-to-camera (flip y and z), velocities rotated by the same flip.

`ImagePrefetcher` replaces the one-random-image-per-step datamanager (data/datamanagers/full_images_datamanager.py:
287-304) for this path: uint8 images stay pinned on the host, image k+1 and its 21 camera floats cross PCIe on a copy
stream while step k renders.  CUDA only.
"""
import json
import math
import os
from typing import Dict, List, Optional

import numpy as np
import torch


# ------------------------------------------------------------------------------------------ transforms.json

def _rotation_between(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """Rotation taking direction a to direction b (Rodrigues; camera_utils.py:449-479), float32 like the reference."""
    a = (a / np.linalg.norm(a)).astype(np.float32)
    b = (b / np.linalg.norm(b)).astype(np.float32)
    v = np.cross(a, b).astype(np.float32)
    eps = 1e-6
    if np.sum(np.abs(v)) < eps:  # parallel: any axis orthogonal to a
        x = np.array([1.0, 0, 0], np.float32) if abs(a[0]) < eps else np.array([0, 1.0, 0], np.float32)
        v = np.cross(a, x).astype(np.float32)
    v = v / np.linalg.norm(v)
    K = np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]], np.float32)
    theta = np.arccos(np.clip(np.dot(a, b), -1, 1)).astype(np.float32)
    return (np.eye(3, dtype=np.float32) + np.sin(theta) * K + (1 - np.cos(theta)) * (K @ K)).astype(np.float32)


def orient_and_center(poses: np.ndarray, method: str = "up", center_method: str = "poses"):
    """(n,4,4) or (n,3,4) camera-to-world -> ((n,3,4) oriented poses, (3,4) transform); camera_utils.py:520-628 for the
    "up" / "none" orientations and the "poses" / "none" centrings."""
    poses = np.asarray(poses, np.float32)
    if poses.shape[-2] == 3:
        bottom = np.tile(np.array([[[0, 0, 0, 1]]], np.float32), (poses.shape[0], 1, 1))
        poses = np.concatenate([poses, bottom], axis=1)
    origins = poses[:, :3, 3]
    if center_method == "poses":
        translation = origins.mean(axis=0)
    elif center_method == "none":
        translation = np.zeros(3, np.float32)
    else:
        raise ValueError(f"unsupported center_method: {center_method}")
    if method == "up":
        up = poses[:, :3, 1].mean(axis=0)
        up = up / np.linalg.norm(up)
        R = _rotation_between(up, np.array([0, 0, 1], np.float32))
    elif method == "none":
        R = np.eye(3, dtype=np.float32)
    else:
        raise ValueError(f"unsupported orientation method: {method}")
    transform = np.concatenate([R, R @ -translation[:, None]], axis=1).astype(np.float32)
    return (transform @ poses).astype(np.float32), transform


def split_indices(n: int, split: str, eval_mode: str = "fraction", train_split_fraction: float = 0.9,
                  eval_interval: int = 8, optimize_eval_cameras: bool = False, filenames: Optional[List[str]] = None):
    """dataparsers_utils.py:23-43 ("fraction"), :46-68 ("filename": basenames containing "train" or "eval", needs
    `filenames`), :69-86 ("interval"), "all".

    optimize_eval_cameras (3dgs-deblur's --optimize-eval-cameras, nerfstudio_dataparser.py:241-252): the train split
    becomes the eval images followed by the training images, and the call returns (indices, detached) with detached[i]
    True for the eval images at the front -- their loss may move only their own camera's pose and velocity rows.  The
    val / test splits keep their order and are all detached, as the reference marks them.  "all" keeps every image
    trained and none detached."""
    i_all = np.arange(n)
    if eval_mode == "fraction":
        n_train = math.ceil(n * train_split_fraction)
        i_train = np.linspace(0, n - 1, n_train, dtype=int)
        i_eval = np.setdiff1d(i_all, i_train)
    elif eval_mode == "filename":
        if filenames is None or len(filenames) != n:
            raise ValueError("eval_mode 'filename' needs the n image filenames")
        i_train, i_eval = [], []
        for i, name in enumerate(filenames):
            base = os.path.basename(name)
            if "train" in base:
                i_train.append(i)
            elif "eval" in base:
                i_eval.append(i)
            else:
                raise ValueError("frame should contain train/eval in its name to use this eval-frame-index eval mode")
        i_train, i_eval = np.array(i_train, dtype=np.int64), np.array(i_eval, dtype=np.int64)
    elif eval_mode == "interval":
        i_train = i_all[i_all % eval_interval != 0]
        i_eval = i_all[i_all % eval_interval == 0]
    elif eval_mode == "all":
        i_train = i_eval = i_all
    else:
        raise ValueError(f"unsupported eval_mode: {eval_mode}")
    detach = optimize_eval_cameras and eval_mode != "all"
    if detach:
        i_train = np.hstack([i_eval, i_train]).ravel().astype(np.int64)
    if split == "train":
        idx = i_train
    elif split in ("val", "test"):
        idx = i_eval
    else:
        raise ValueError(f"Unknown dataparser split {split}")
    if not optimize_eval_cameras:
        return idx
    detached = np.zeros(len(idx), bool)
    if detach:  # the reference's rule, position < len(i_eval), in either split (val / test: all of them)
        detached[:len(i_eval)] = True
    return idx, detached


def _auto_downscale(data_dir: str, rel_path: str) -> int:
    """The reference's rule (nerfstudio_dataparser.py:508-523): halve while max(h, w) > 1600 px AND the next
    `images_<2^k>` folder holds the file."""
    from PIL import Image

    with Image.open(os.path.join(data_dir, rel_path)) as im:
        w, h = im.size
    df = 0
    while max(h, w) / 2 ** df > 1600 and os.path.exists(
            os.path.join(data_dir, f"images_{2 ** (df + 1)}", os.path.basename(rel_path))):
        df += 1
    return 2 ** df


def load_transforms(path: str, split: str = "train", *, scale_factor: float = 1.0, downscale_factor: Optional[int] = None,
                    orientation_method: str = "up", center_method: str = "poses", auto_scale_poses: bool = True,
                    eval_mode: str = "fraction", train_split_fraction: float = 0.9, eval_interval: int = 8,
                    optimize_eval_cameras: bool = False) -> Dict:
    """Parse a nerfstudio dataset directory (or its transforms.json) the way the reference's dataparser does.

    Returns a dict: image_filenames (list), camera_to_worlds (n,3,4) f32, fx, fy, cx, cy (n,) f32, height, width (n,) i64,
    velocities (n,6) f32 or None (linear part already in scene units), exposure_time, rolling_shutter_time (floats or
    None), dataparser_scale (float), dataparser_transform (3,4) f32, indices (n,) into the name-sorted frame list, and
    detached: None, or with optimize_eval_cameras a bool (n,) marking the eval images split_indices put at the front of
    the train split (pass their positions as PipelinedTrainer(detached_cameras=...)).  A dataset that lists its split
    files ("<split>_filenames") cannot optimise its eval cameras (AssertionError, as the reference asserts)."""
    if path.endswith(".json"):
        meta_path, data_dir = path, os.path.dirname(path)
    else:
        meta_path, data_dir = os.path.join(path, "transforms.json"), path
    with open(meta_path, "r", encoding="utf-8") as f:
        meta = json.load(f)
    frames = meta["frames"]
    if not frames:
        raise ValueError("transforms.json has no frames")

    def fname(rel, df):
        rel = rel.replace("\\", "/")
        if df > 1:
            return os.path.join(data_dir, f"images_{df}", os.path.basename(rel))
        return os.path.join(data_dir, rel)

    if downscale_factor is None:
        downscale_factor = _auto_downscale(data_dir, frames[0]["file_path"])
    names = [fname(fr["file_path"], downscale_factor) for fr in frames]
    order = np.argsort(names)
    frames = [frames[i] for i in order]
    names = [names[i] for i in order]

    def per_camera(key, cast):
        if key in meta:
            return np.full(len(frames), cast(meta[key]))
        missing = [i for i, fr in enumerate(frames) if key not in fr]
        if missing:
            raise AssertionError(f"{key} not specified in frame")
        return np.array([cast(fr[key]) for fr in frames])

    fx, fy = per_camera("fl_x", float), per_camera("fl_y", float)
    cx, cy = per_camera("cx", float), per_camera("cy", float)
    height, width = per_camera("h", int), per_camera("w", int)

    velocities = None
    if any("camera_linear_velocity" in fr for fr in frames):
        rows = []
        for fr in frames:
            if "camera_linear_velocity" not in fr or "camera_angular_velocity" not in fr:
                raise AssertionError("camera velocities must be given for every frame or for none")
            row = list(fr["camera_linear_velocity"]) + list(fr["camera_angular_velocity"])
            if len(row) != 6:
                raise AssertionError("camera velocities must have 3 + 3 components")
            rows.append(row)
        velocities = np.array(rows).astype(np.float32)

    orientation_method = meta.get("orientation_override", orientation_method)
    auto_scale_poses = meta.get("auto_scale_poses_override", auto_scale_poses)
    poses = np.array([fr["transform_matrix"] for fr in frames]).astype(np.float32)
    poses, transform = orient_and_center(poses, orientation_method, center_method)
    scale = 1.0
    if auto_scale_poses:
        scale /= float(np.max(np.abs(poses[:, :3, 3])))
    scale *= scale_factor
    poses[:, :3, 3] *= scale

    split_key = f"{split}_filenames"
    detached = None
    if split_key in meta:
        if optimize_eval_cameras:
            raise AssertionError("optimize_eval_cameras needs a split rule, not listed <split>_filenames")
        wanted = {fname(x, downscale_factor) for x in meta[split_key]}
        unmatched = wanted.difference(names)
        if unmatched:
            raise RuntimeError(f"Some filenames for split {split} were not found: {unmatched}.")
        idx = np.array([i for i, nme in enumerate(names) if nme in wanted], dtype=np.int64)
    elif any(f"{s}_filenames" in meta for s in ("train", "val", "test")):
        raise RuntimeError(f"The dataset's list of filenames for split {split} is missing.")
    else:
        idx = split_indices(len(names), split, eval_mode, train_split_fraction, eval_interval, optimize_eval_cameras, names)
        if optimize_eval_cameras:
            idx, detached = idx
        idx = idx.astype(np.int64)

    if velocities is not None:
        velocities = velocities[idx].copy()
        velocities[:, :3] *= scale  # :336 (the literal reads scale_factor: the combined pose scale at that point)
    if "applied_scale" in meta:
        scale_out = scale * float(meta["applied_scale"])
    else:
        scale_out = scale
    if "applied_transform" in meta:
        at = np.concatenate([np.array(meta["applied_transform"], np.float32), np.array([[0, 0, 0, 1]], np.float32)], 0)
        transform_out = (transform @ at).astype(np.float32)
    else:
        transform_out = transform

    s = 1.0 / downscale_factor  # Cameras.rescale_output_resolution(1 / downscale_factor), floor on the sizes
    f32 = lambda a: (np.asarray(a, np.float32)[idx] * np.float32(s)).astype(np.float32)
    size = lambda a: np.floor(np.asarray(a, np.float64)[idx] * s).astype(np.int64)
    return dict(
        image_filenames=[names[i] for i in idx], camera_to_worlds=poses[idx][:, :3, :4].copy(),
        fx=f32(fx), fy=f32(fy), cx=f32(cx), cy=f32(cy), height=size(height), width=size(width),
        velocities=velocities, exposure_time=meta.get("exposure_time"), rolling_shutter_time=meta.get("rolling_shutter_time"),
        dataparser_scale=scale_out, dataparser_transform=transform_out, indices=idx, detached=detached)


_PLY_TYPES = {"char": "i1", "uchar": "u1", "int8": "i1", "uint8": "u1", "short": "i2", "ushort": "u2", "int16": "i2",
              "uint16": "u2", "int": "i4", "uint": "u4", "int32": "i4", "uint32": "u4", "float": "f4", "float32": "f4",
              "double": "f8", "float64": "f8"}


def load_ply_points(path: str, dataparser_transform=None, dataparser_scale: float = 1.0):
    """Seed point cloud (`sparse_pc.ply`, `ply_file_path` in transforms.json) -> (xyz (n,3) f32, rgb (n,3) u8), moved
    into the dataparser's output frame like nerfstudio_dataparser.py:469-491 does: [xyz 1] @ transform^T, then * scale.
    Reads ascii and binary_little_endian vertex elements with x, y, z (+ red, green, blue); no external PLY library."""
    with open(path, "rb") as f:
        if f.readline().strip() != b"ply":
            raise ValueError("not a PLY file")
        fmt, n_vertex, props, in_vertex = None, 0, [], False
        while True:
            line = f.readline()
            if not line:
                raise ValueError("PLY header without end_header")
            tok = line.decode("ascii", "replace").split()
            if not tok:
                continue
            if tok[0] == "format":
                fmt = tok[1]
            elif tok[0] == "element":
                in_vertex = tok[1] == "vertex"
                if in_vertex:
                    n_vertex = int(tok[2])
                elif n_vertex and not props:
                    raise ValueError("PLY vertex element without properties")
            elif tok[0] == "property" and in_vertex:
                if tok[1] == "list":
                    raise ValueError("list properties on vertices are not supported")
                props.append((tok[2], _PLY_TYPES[tok[1]]))
            elif tok[0] == "end_header":
                break
        names = [nme for nme, _ in props]
        if not all(k in names for k in ("x", "y", "z")):
            raise ValueError("PLY vertices need x, y, z")
        if fmt == "ascii":
            rows = np.loadtxt(f, max_rows=n_vertex, ndmin=2)
            cols = {nme: rows[:, i] for i, nme in enumerate(names)}
        elif fmt == "binary_little_endian":
            dt = np.dtype([(nme, "<" + t) for nme, t in props])
            data = np.frombuffer(f.read(dt.itemsize * n_vertex), dtype=dt, count=n_vertex)
            cols = {nme: data[nme] for nme in names}
        else:
            raise ValueError(f"unsupported PLY format: {fmt}")
    xyz = np.stack([cols["x"], cols["y"], cols["z"]], axis=1).astype(np.float32)
    if all(k in cols for k in ("red", "green", "blue")):
        rgb = np.stack([cols["red"], cols["green"], cols["blue"]], axis=1)
        if rgb.dtype.kind == "f" and rgb.max(initial=0) <= 1.0:
            rgb = rgb * 255
        rgb = rgb.astype(np.uint8)
    else:
        rgb = np.full((xyz.shape[0], 3), 128, np.uint8)
    if dataparser_transform is not None:
        T = np.asarray(dataparser_transform, np.float32)
        xyz = (np.concatenate([xyz, np.ones_like(xyz[:, :1])], axis=1) @ T.T).astype(np.float32)
    xyz = xyz * np.float32(dataparser_scale)
    return xyz, rgb


def load_image_u8(path: str, alpha_color=None) -> torch.Tensor:
    """One training image as an (H, W, 3) or (H, W, 4) uint8 tensor, the way the reference's dataset reads it
    (nerfstudio/data/datasets/base_dataset.py:61-79, 95-110): greyscale is repeated to three channels; with `alpha_color`
    (three floats in [0, 1]) an RGBA image is composited over that colour and comes back with three channels, otherwise
    the alpha channel is kept for the model to composite against its own background (splatfacto.py:912-923)."""
    from PIL import Image

    with Image.open(path) as im:
        a = np.array(im, dtype="uint8")
    if a.ndim == 2:
        a = np.repeat(a[:, :, None], 3, axis=2)
    if a.ndim != 3 or a.shape[2] not in (3, 4):
        raise ValueError(f"Image shape of {a.shape} is incorrect.")
    img = torch.from_numpy(a)
    if alpha_color is not None and img.shape[-1] == 4:
        col = torch.as_tensor(alpha_color, dtype=torch.float32)
        if not bool(((col >= 0) & (col <= 1)).all()):
            raise ValueError("alpha color given is out of range between [0, 1].")
        alpha = img[:, :, -1:] / 255.0
        img = torch.clamp(img[:, :, :3] * alpha + 255.0 * col * (1.0 - alpha), min=0, max=255).to(torch.uint8)
    return img.contiguous()


def composite_u8(image_u8: torch.Tensor, background: torch.Tensor) -> torch.Tensor:
    """Float target image in [0, 1] from a uint8 image; an alpha channel is composited over `background` (3 floats)
    like Splatfacto does per step (splatfacto.py:900-923): alpha * rgb + (1 - alpha) * background."""
    img = image_u8.float() / 255.0
    if img.shape[2] == 4:
        alpha = img[..., -1:]
        return alpha * img[..., :3] + (1 - alpha) * background
    return img


def to_gsplat_camera(camera_to_world, velocity=None) -> Dict[str, torch.Tensor]:
    """OpenGL camera-to-world (3,4) [+ camera-frame velocity (6,)] -> what the gsplat operators take
    (splatfacto.py:733-747: R <- R diag(1,-1,-1), viewmat = [R^T | -R^T t]; :799-800: velocities rotated by the flip)."""
    c2w = torch.as_tensor(camera_to_world, dtype=torch.float32)
    flip = torch.tensor([1.0, -1.0, -1.0])
    R = c2w[:3, :3] * flip[None, :]  # R @ diag(flip)
    t = c2w[:3, 3]
    viewmat = torch.eye(4)
    viewmat[:3, :3] = R.T
    viewmat[:3, 3] = -(R.T @ t)
    out = dict(viewmat=viewmat, cam_pos=t.clone())
    if velocity is not None:
        v = torch.as_tensor(velocity, dtype=torch.float32)
        out["lin_vel"], out["ang_vel"] = flip * v[:3], flip * v[3:]
    return out


# ------------------------------------------------------------------------------------------ per-image dispatcher

class ImagePrefetcher:
    """Double-buffered H2D prefetch of (uint8 image, camera floats) pairs on a copy stream.

    images: list of (H, W, 3) uint8 host tensors (pinned here if they are not); cameras: list of 1-D float32 host tensors
    (viewmat 12 | lin_vel 3 | ang_vel 3 | cam_pos 3 in bench.py's layout; any fixed length works).  Usage:

        pf = ImagePrefetcher(images, cameras, device); pf.start(order[0])
        for k in range(steps):
            img_u8, cam = pf.get(next_index=order[k + 1])   # waits for copy k on the compute stream, queues copy k+1
            ... train step on img_u8.float() / 255 and cam ...
            pf.done()                                        # the buffers of step k may be overwritten again
    """

    def __init__(self, images: List[torch.Tensor], cameras: List[torch.Tensor], device):
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("ImagePrefetcher needs a CUDA device (there is no CPU path)")
        if len(images) != len(cameras) or not images:
            raise ValueError("need one camera vector per image")
        shape, n_cam = tuple(images[0].shape), cameras[0].numel()
        for im, cam in zip(images, cameras):
            if im.dtype != torch.uint8 or tuple(im.shape) != shape or cam.dtype != torch.float32 or cam.numel() != n_cam:
                raise ValueError("all images must be uint8 of one shape, all cameras float32 of one length")
        self.images = [im if im.is_pinned() else im.contiguous().pin_memory() for im in images]
        self.cameras = [c if c.is_pinned() else c.contiguous().pin_memory() for c in cameras]
        self.device = device
        self.copy_stream = torch.cuda.Stream(device=device)
        self.buf_img = [torch.empty(shape, dtype=torch.uint8, device=device) for _ in range(2)]
        self.buf_cam = [torch.empty(n_cam, dtype=torch.float32, device=device) for _ in range(2)]
        self.ready = [torch.cuda.Event() for _ in range(2)]
        self.consumed = [torch.cuda.Event() for _ in range(2)]
        self.bytes_per_step = self.images[0].numel() + 4 * n_cam
        self._k = 0
        self._started = False

    def _queue(self, slot: int, index: int):
        with torch.cuda.stream(self.copy_stream):
            self.copy_stream.wait_event(self.consumed[slot])
            self.buf_img[slot].copy_(self.images[index], non_blocking=True)
            self.buf_cam[slot].copy_(self.cameras[index], non_blocking=True)
            self.ready[slot].record(self.copy_stream)

    def start(self, first_index: int):
        main = torch.cuda.current_stream(self.device)
        for s in range(2):
            self.consumed[s].record(main)
        self._k = 0
        self._queue(0, first_index)
        self._started = True

    def get(self, next_index: Optional[int] = None):
        if not self._started:
            raise RuntimeError("call start() first")
        slot = self._k % 2
        torch.cuda.current_stream(self.device).wait_event(self.ready[slot])
        if next_index is not None:
            self._queue(1 - slot, next_index)
        return self.buf_img[slot], self.buf_cam[slot]

    def done(self):
        self.consumed[self._k % 2].record(torch.cuda.current_stream(self.device))
        self._k += 1
