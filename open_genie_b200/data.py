"""Data path — mirrors genie/module/data.py:24-233 (LightningDataset, Platformer2D) and genie/dataset.py:95-161
(LightningPlatformer2D): same constructors, same `from_config`, same loaders, same tensors.

GPU-first change (opt-in, `raw_uint8=True` + VideoBatchPrefetcher): the reference converts every decoded frame to
fp32, divides by 255 and rearranges on the CPU workers, then ships 4 bytes per element over PCIe. Here the workers hand
over the frames exactly as OpenCV decodes them (uint8, t h w c, BGR); batches are staged in pinned memory, copied on a
side stream while the previous step computes, and ONE kernel (og_frames_u8_to_video) does the colour swap, the /255 and
the layout change on the device — 1/4 of the H2D bytes and no per-frame CPU float work. The default
(`raw_uint8=False`) reproduces the reference's CPU tensors bit for bit.
"""
from __future__ import annotations

from os import listdir, path
from random import randint
from typing import Callable, Iterable, Iterator

import torch
from torch import Tensor
from torch.utils.data import DataLoader, Dataset, IterableDataset

from .utils import default, exists

try:  # pragma: no cover - depends on the environment
    from lightning import LightningDataModule  # type: ignore
except Exception:
    class LightningDataModule:                  # minimal stand-in (lightning is not installed in the build image)
        def __init__(self, *a, **k):
            pass

        def save_hyperparameters(self, *a, **k):
            pass


def default_iterdata_worker_init(worker_id: int) -> None:
    """genie/utils.py:61-74: split an IterableDataset's [start, end) range across DataLoader workers."""
    import math
    info = torch.utils.data.get_worker_info()
    if info is None:
        return
    ds = info.dataset
    if not hasattr(ds, 'start') or not hasattr(ds, 'end'):
        return
    per_worker = int(math.ceil((ds.end - ds.start) / float(info.num_workers)))
    ds.start = ds.start + worker_id * per_worker
    ds.end = min(ds.start + per_worker, ds.end)


class LightningDataset(LightningDataModule):
    """Abstract data module — genie/module/data.py:24-137."""

    @classmethod
    def from_config(cls, conf_path: str, *args, key: str = 'dataset') -> 'LightningDataset':
        import yaml
        with open(conf_path, 'r') as f:
            conf = yaml.safe_load(f)
        return cls(*args, **conf[key])

    def __init__(self, *args, batch_size: int = 16, num_workers: int = 0, train_shuffle: bool | None = None,
                 val_shuffle: bool | None = None, val_batch_size: None | int = None, worker_init_fn: None | Callable = None,
                 collate_fn: None | Callable = None, train_sampler: None | Callable = None,
                 val_sampler: None | Callable = None, test_sampler: None | Callable = None) -> None:
        super().__init__()
        self.train_dataset = None
        self.valid_dataset = None
        self.test__dataset = None
        self.num_workers = num_workers
        self.batch_size = batch_size
        self.train_shuffle = train_shuffle
        self.val_shuffle = val_shuffle
        self.train_sampler = train_sampler
        self.valid_sampler = val_sampler
        self.test__sampler = test_sampler
        self.collate_fn = collate_fn
        self.worker_init_fn = worker_init_fn
        self.val_batch_size = default(val_batch_size, batch_size)

    def setup(self, stage: str) -> None:
        raise NotImplementedError('This is an abstract datamodule class. You should use one of the concrete '
                                  'subclasses that represents an actual dataset.')

    def _loader(self, dataset, sampler, batch_size, shuffle) -> DataLoader:
        worker_init_fn = self.worker_init_fn
        if isinstance(self.train_dataset, IterableDataset):
            worker_init_fn = default(self.worker_init_fn, default_iterdata_worker_init)
        return DataLoader(dataset, sampler=sampler, batch_size=batch_size, shuffle=shuffle, collate_fn=self.collate_fn,
                          num_workers=self.num_workers, worker_init_fn=worker_init_fn)

    def train_dataloader(self) -> DataLoader:
        return self._loader(self.train_dataset, self.train_sampler, self.batch_size, self.train_shuffle)

    def val_dataloader(self) -> DataLoader:
        return self._loader(self.valid_dataset, self.valid_sampler, self.val_batch_size, self.val_shuffle)

    def test_dataloader(self) -> DataLoader:
        return self._loader(self.test__dataset, self.test__sampler, self.val_batch_size, self.val_shuffle)


class Platformer2D(Dataset):
    """mp4 clips recorded from the Procgen platformers — genie/module/data.py:139-233. `raw_uint8=True` returns the
    decoded frames untouched (uint8, (t, h, w, c), BGR) for the device-side decode of VideoBatchPrefetcher."""

    def __init__(self, root: str, split: str = 'train', env_name: str = 'Coinrun', padding: str = 'none',
                 randomize: bool = False, transform: Callable | None = None, num_frames: int = 16,
                 output_format: str = 't c h w', raw_uint8: bool = False) -> None:
        super().__init__()
        self.root = path.join(root, env_name, split)
        self.split = split
        self.padding = padding
        self.randomize = randomize
        self.num_frames = num_frames
        self.output_format = output_format
        self.transform = transform if exists(transform) else (lambda x: x)
        self.raw_uint8 = raw_uint8
        self.file_names = [path.join(self.root, f) for f in listdir(self.root)]

    def __len__(self) -> int:
        return len(self.file_names)

    def __getitem__(self, idx: int) -> Tensor:
        return self.load_video_slice(self.file_names[idx], self.num_frames, None if self.randomize else 0)

    def load_video_slice(self, video_path: str, num_frames: int, start_frame: int | None = None) -> Tensor:
        import cv2
        cap = cv2.VideoCapture(video_path)
        total_frames = int(cap.get(cv2.CAP_PROP_FRAME_COUNT))
        num_frames = min(num_frames, total_frames)              # shorter videos are returned whole (data.py:191-193)
        start_frame = start_frame if exists(start_frame) else randint(0, total_frames - num_frames)
        cap.set(cv2.CAP_PROP_POS_FRAMES, start_frame)
        frames = []
        for _ in range(num_frames):
            ret, frame = cap.read()
            if ret:
                if not self.raw_uint8:
                    frame = cv2.cvtColor(frame, cv2.COLOR_BGR2RGB)
                frames.append(torch.from_numpy(frame))
            else:                                                # end of video: padding policy (data.py:207-227)
                missing = num_frames - len(frames)
                match self.padding:
                    case 'none':
                        pass
                    case 'repeat':
                        frames.extend([frames[-1]] * missing)
                    case 'zero':
                        frames.extend([torch.zeros_like(frames[-1])] * missing)
                    case 'random':   # (the reference's torch.rand_like on a uint8 frame raises; the evident intent: noise frames)
                        frames.extend([torch.randint(0, 256, frames[-1].shape, dtype=torch.uint8)] * missing)
                    case _:
                        raise ValueError(f'Invalid padding type: {self.padding}')
                break
        cap.release()
        if self.raw_uint8:
            return torch.stack(frames)
        video = torch.stack(frames) / 255.
        video = _rearrange_thwc(video, self.output_format)
        return self.transform(video)


def _rearrange_thwc(video: Tensor, output_format: str) -> Tensor:
    """einops.rearrange(video, f't h w c -> {output_format}') for the permutations the reference uses."""
    src = ['t', 'h', 'w', 'c']
    dst = output_format.split()
    if sorted(dst) != sorted(src):
        raise ValueError(f'Invalid output format: {output_format!r}')
    return video.permute(*[src.index(a) for a in dst]).contiguous()


class LightningPlatformer2D(LightningDataset):
    """genie/dataset.py:95-161."""

    def __init__(self, root, env_name: str = 'Coinrun', padding: str = 'none', randomize: bool = False,
                 transform: Callable | None = None, num_frames: int = 16, output_format: str = 't c h w',
                 raw_uint8: bool = False, **kwargs) -> None:
        super().__init__(**kwargs)
        self.root = root
        self.padding = padding
        self.env_name = env_name
        self.transform = transform
        self.randomize = randomize
        self.num_frames = num_frames
        self.output_format = output_format
        self.raw_uint8 = raw_uint8
        self.save_hyperparameters()

    def _make(self, split: str) -> Platformer2D:
        return Platformer2D(root=self.root, split=split, padding=self.padding, env_name=self.env_name,
                            transform=self.transform, randomize=self.randomize, num_frames=self.num_frames,
                            output_format=self.output_format, raw_uint8=self.raw_uint8)

    def setup(self, stage: str) -> None:
        match stage:
            case 'fit':
                self.train_dataset = self._make('train')
                self.valid_dataset = self._make('val')
            case 'test':
                self.test__dataset = self._make('test')
            case _:
                raise ValueError(f'Invalid stage: {stage}')


def frames_to_video(frames_u8: Tensor, bgr: bool = True, internal: bool = False, cpad: int = 3) -> Tensor:
    """uint8 (N, T, H, W, 3) frames ON THE DEVICE -> (N, 3, T, H, W) video in [0, 1]: fp32 NCDHW (reference format), or
    with `internal=True` the bf16 NDHWC activation format (channel pitch `cpad`, zero padded)."""
    from . import _lib, ops
    ops._require_cuda(frames_u8, 'frames')
    if frames_u8.dtype != torch.uint8 or frames_u8.dim() != 5 or frames_u8.shape[-1] != 3:
        raise ValueError(f'expected uint8 frames of shape (N, T, H, W, 3), got {frames_u8.dtype} {tuple(frames_u8.shape)}')
    f = frames_u8.contiguous()
    N, T, H, W, _ = f.shape
    if internal:
        out = torch.empty((N, T, H, W, cpad), dtype=torch.bfloat16, device=f.device)
        _lib.call('og_frames_u8_to_video', f.data_ptr(), int(bgr), out.data_ptr(), 1, cpad, N, T, H, W, ops._stream())
        return out.permute(0, 4, 1, 2, 3)[:, :3]
    out = torch.empty((N, 3, T, H, W), dtype=torch.float32, device=f.device)
    _lib.call('og_frames_u8_to_video', f.data_ptr(), int(bgr), out.data_ptr(), 0, 3, N, T, H, W, ops._stream())
    return out


class VideoBatchPrefetcher:
    """Wraps a DataLoader over a `raw_uint8=True` dataset: yields (N, 3, T, H, W) fp32 videos in [0, 1] that are already
    on the device. Two pinned staging buffers and a copy stream: batch k+1 crosses PCIe (1 byte per element) and is
    decoded by og_frames_u8_to_video while the consumer's kernels of batch k run on the main stream."""

    def __init__(self, loader: Iterable, device='cuda', bgr: bool = True, internal: bool = False):
        self.loader, self.device, self.bgr, self.internal = loader, torch.device(device), bgr, internal
        self.stream = torch.cuda.Stream(device=self.device)
        self._pinned = [None, None]
        self._inflight = [None, None]      # event after which a staging buffer's last H2D copy has completed
        self.h2d_bytes = 0

    def __len__(self):
        return len(self.loader)

    def _stage(self, batch: Tensor, slot: int):
        if batch.dtype != torch.uint8:
            raise ValueError('VideoBatchPrefetcher needs uint8 frames: build the dataset with raw_uint8=True')
        if self._inflight[slot] is not None:
            self._inflight[slot].synchronize()      # the GPU may lag: do not overwrite a buffer whose copy is still in flight
        buf = self._pinned[slot]
        if buf is None or buf.shape != batch.shape:
            buf = torch.empty(batch.shape, dtype=torch.uint8).pin_memory()
            self._pinned[slot] = buf
        buf.copy_(batch)
        self.h2d_bytes += buf.numel()
        with torch.cuda.stream(self.stream):
            dev = buf.to(self.device, non_blocking=True)
            copied = torch.cuda.Event()
            copied.record(self.stream)
            self._inflight[slot] = copied
            video = frames_to_video(dev, self.bgr, self.internal)
            ev = torch.cuda.Event()
            ev.record(self.stream)
        return video, dev, ev

    def __iter__(self) -> Iterator[Tensor]:
        it = iter(self.loader)
        slot = 0
        try:
            nxt = self._stage(next(it), slot)
        except StopIteration:
            return
        while nxt is not None:
            video, raw, ev = nxt
            slot ^= 1
            try:
                nxt = self._stage(next(it), slot)      # overlaps with the consumer's work on `video`
            except StopIteration:
                nxt = None
            torch.cuda.current_stream(self.device).wait_event(ev)
            video.record_stream(torch.cuda.current_stream(self.device))
            yield video
