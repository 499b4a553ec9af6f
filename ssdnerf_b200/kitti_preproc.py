"""`python -m ssdnerf_b200.kitti_preproc --kitti-dir --out-dir --out-size --out-border`: the reference's tools/kitti_preproc.py on the
GPU (see ssdnerf_b200/kitti.py)."""
from .kitti import main

if __name__ == '__main__':
    main()
