"""Writes the data-path test vectors: tests/golden/platformer/Coinrun/{train,val,test}/clip*.mp4 (64 x 64 frames of 8 x 8
colour blocks; clip0 of each split is shorter than 16 frames) and tests/golden/data_path.json, the SHA-256 digests of what
the reference's own Platformer2D returns for them (every output format x padding mode of the train split).

    python oracle/make_golden_data_path.py /path/to/open-genie     # a checkout of the reference project
"""
import json
import os
import shutil
import sys
from pathlib import Path

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLIPS = os.path.join(ROOT, 'tests', 'golden', 'platformer')


def write_clips(root):
    import cv2
    rng = np.random.default_rng(0)
    for split, n in (('train', 5), ('val', 2), ('test', 2)):
        d = root / 'Coinrun' / split
        d.mkdir(parents=True)
        for i in range(n):
            w = cv2.VideoWriter(str(d / f'clip{i}.mp4'), cv2.VideoWriter_fourcc(*'mp4v'), 15, (64, 64))
            assert w.isOpened()
            base = rng.integers(0, 255, (8, 8, 3))
            for t in range(12 if i == 0 else 20):
                frame = np.kron((base + 9 * t) % 256, np.ones((8, 8, 1))).astype(np.uint8)
                w.write(frame)
            w.release()


def main(ref_root):
    sys.path[:0] = [os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'oracle', '_shim'), ref_root]
    from test_data_path import digest
    from genie.module.data import Platformer2D
    shutil.rmtree(CLIPS, ignore_errors=True)
    write_clips(Path(CLIPS))
    out = {}
    for fmt in ('t c h w', 'c t h w'):
        for padding in ('none', 'repeat', 'zero'):
            ds = Platformer2D(CLIPS, split='train', padding=padding, num_frames=16, output_format=fmt)
            items = [ds[i] for i in range(len(ds))]
            out[f'{fmt}|{padding}'] = {'file_names': [os.path.basename(n) for n in ds.file_names],
                                       'shapes': [list(t.shape) for t in items],
                                       'sha256': [digest(t) for t in items]}
    with open(os.path.join(ROOT, 'tests', 'golden', 'data_path.json'), 'w') as f:
        json.dump(out, f, indent=1)


if __name__ == '__main__':
    main(sys.argv[1])
