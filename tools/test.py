"""Dataset evaluation with the reference's command line (its tools/test.py); the logic is patchfusion_b200/evaluate.py.

    python tools/test.py <config.py> --ckp-path <ckpt> --cai-mode m1 --test-type normal --work-dir <dir> \
        --image-raw-shape 2160 3840 --patch-split-num 4 4 [--save] [--cfg-options k=v ...]
    torchrun --nproc-per-node 8 tools/test.py <config.py> ... --launcher pytorch
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from patchfusion_b200.evaluate import main  # noqa: E402

if __name__ == '__main__':
    main()
