"""The host restatement of the top-k order (tests/topk_oracle.py) against torch.sort(descending=True, stable=True), the
order the contract names, on matrices full of ties and special values.  No GPU needed."""
import numpy as np
import torch

from topk_oracle import order_image, topk


def _special(rng, b, n):
    pool = np.array([np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, 1.0, -1.0, 0.5, 1e-40, -1e-40], np.float32)
    m = pool[rng.integers(0, len(pool), (b, n))]
    m[0] = 3.0  # an all-equal row
    return m


def test_order_image_is_monotone():
    v = np.array([-np.inf, -3.0, -1e-40, -0.0, 0.0, 1e-40, 2.0, np.inf, np.nan], np.float32)
    img = order_image(v).astype(np.int64)
    assert (np.diff(img) >= 0).all() and img[3] == img[4]
    assert (np.diff(img[[0, 1, 2, 3, 5, 6, 7, 8]]) > 0).all()


def test_topk_matches_stable_descending_sort():
    rng = np.random.default_rng(3)
    for b, n in ((5, 1), (7, 33), (4, 300)):
        m = _special(rng, b, n)
        for k in (1, 3, n, n + 5):
            pos, val = topk(m, k)
            ref = torch.sort(torch.from_numpy(m), dim=1, descending=True, stable=True).indices.numpy()[:, :k]
            kk = min(k, n)
            assert (pos[:, :kk] == ref).all()
            assert (pos[:, kk:] == -1).all() and np.isneginf(val[:, kk:]).all()
            got = val[:, :kk].view(np.uint32)
            assert (got == np.take_along_axis(m, ref, 1).view(np.uint32)).all()  # raw values, bit for bit


def test_topk_exclude():
    rng = np.random.default_rng(4)
    m = rng.integers(-2, 3, (6, 40)).astype(np.float32)
    ex = [rng.choice(60, 30, replace=False) - 10 for _ in range(6)]  # some positions out of range
    pos, _ = topk(m, 40, ex)
    for i in range(6):
        keep = [p for p in pos[i] if p >= 0]
        assert not set(keep) & set(ex[i].tolist())
        assert len(keep) == 40 - len([p for p in ex[i] if 0 <= p < 40])
