"""Seeded inputs of the reference comparisons (tests/test_oracle_golden.py, make_reference_vectors.py): one definition for both."""
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
FCLAYER_ENCS = [1, 2, 4, 12, 16, 20, 36, 64, 3]
WHOLE_MODELS = ["fc", "cnn", "cnn_48", "binary160", "ternary64", "rand_fp130_64", "rand_nf4_64", "1k"]


def load(name):
    from bitnetmcu_b200.model import Model
    return Model.load(os.path.join(HERE, "models", name + ".bnm"))


def fclayer_cases(encs=FCLAYER_ENCS):
    for enc in encs:
        rng = np.random.default_rng(enc)
        for n_in, n_out in [(256, 64), (64, 10), (160, 160), (320, 7)]:
            if enc == 64:
                n_in = (n_in + 9) // 10 * 10
                w = rng.integers(0, 65536, size=n_out * n_in // 10, dtype=np.uint32).astype(np.uint16)
            else:
                w = rng.integers(0, 2 ** 32, size=n_out * n_in // 4 + 4, dtype=np.uint64).astype(np.uint32)
            act = rng.integers(-128, 128, size=n_in + 16).astype(np.int8)
            yield f"{enc}_{n_in}_{n_out}", (act, w, enc, n_in, n_out)


def relunorm_cases():
    rng = np.random.default_rng(7)
    for trial in range(300):
        n = int(rng.integers(1, 300))
        scale = int(rng.choice([1, 100, 20000, 500000, 4000000]))
        x = rng.integers(-scale, scale + 1, size=n).astype(np.int32)
        if trial % 7 == 0:
            x = -np.abs(x) - 1
        if trial % 11 == 0:
            x[rng.integers(0, n)] = 2 ** (7 + trial % 20) - 1
        yield str(trial), x


def conv_pool_cases():
    rng = np.random.default_rng(9)
    for xy in (16, 14, 6, 4, 3):
        for i in range(20):
            act = rng.integers(-20000, 20000, size=xy * xy).astype(np.int32)
            w = rng.integers(-128, 128, size=9).astype(np.int8)
            yield f"{xy}_{i}", (act, w, xy)


def whole_model_images(m):
    from bitnetmcu_b200 import model as M
    rng = np.random.default_rng(11)
    n = 3000 if m.model_class == M.MODEL_FCMNIST else 600
    imgs = rng.integers(-128, 128, size=(n, 256)).astype(np.int8)
    imgs[:50] = np.clip(imgs[:50], -20, 127)          # MNIST-like background
    imgs[50:60] = -128
    imgs[60:70] = 127
    imgs[70:80] = 0
    return imgs
