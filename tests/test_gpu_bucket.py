"""The owner-computes gradient of the replaced entities (kge_train_bucket.cu) against the atomic scatter it replaces
(KGE_B200_TRAIN_REPL=scatter), on the same inputs: the forward pass is the same kernel, so scores are bit-equal; every
g * Q term is formed with the same fp32 operations, so the gradients differ only in the order of the additions."""
import numpy as np
import pytest
import torch

from ampligraph_b200 import _lib

pytestmark = pytest.mark.gpu


def _engine(*a, **kw):
    from ampligraph_b200.engine import KGEEngine
    return KGEEngine(*a, **kw)


def _tables(model, E, R, k, rng, scale=0.3):
    K = k if model == "DistMult" else 2 * k
    return rng.uniform(-scale, scale, (E, K)).astype(np.float32), rng.uniform(-scale, scale, (R, K)).astype(np.float32)


def _zipf_triples(E, R, n, rng):
    w = 1.0 / np.arange(1, E + 1)
    cdf = np.cumsum(w / w.sum())
    perm = rng.permutation(E)
    s, o = perm[np.searchsorted(cdf, rng.random(n))], perm[np.searchsorted(cdf, rng.random(n))]
    return np.stack([s, rng.integers(0, R, n), o], 1).astype(np.int32)


def _dev(a):
    return torch.as_tensor(a).cuda().contiguous()


def _close(a, b, rtol):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max() <= rtol * max(np.abs(b).max(), 1e-30) + 1e-7


def _bucketed_entries(eng, B):
    """Entries the bucket pre-pass placed in the last step (offset[n_ent] of the workspace's CSR)."""
    ws = eng._train_ws.view(torch.int32)
    off0 = (4 * eng.n_ent + 15) // 16 * 4
    return int(ws[off0 + eng.n_ent].item())


def _run(path, model, k, eta, E, R, t, negatives, monkeypatch, steps=1, mode=_lib.STEP_FUSED, ext=None, seed=3):
    monkeypatch.setenv("KGE_B200_TRAIN_REPL", path)
    rng = np.random.default_rng(5)
    ent, rel = _tables(model, E, R, k, rng)
    B = t.shape[0]
    eng = _engine(model, k, eta, E, R, loss="self_adversarial", optimizer="sgd", optimizer_params={"learning_rate": 1e-3})
    eng.set_embeddings(ent, rel)
    sp = torch.empty(B, device="cuda"); sn = torch.empty(eta * B, device="cuda")
    neg = tuple(_dev(x) for x in negatives) if negatives is not None else None
    out = []
    for step in range(steps):
        kw = dict(scores_pos=sp, scores_neg=sn) if mode == _lib.STEP_FUSED else dict(dpos=_dev(ext[0]), dneg=_dev(ext[1]))
        eng.forward_backward(_dev(t), neg, seed=seed, step=step, mode=mode, **kw)
        torch.cuda.synchronize()
        if step == 0:
            out += [sp.cpu().numpy().copy(), sn.cpu().numpy().copy(), eng.g_ent.cpu().numpy().copy(), eng.g_rel.cpu().numpy().copy()]
            if path == "gather":
                assert _bucketed_entries(eng, B) == eta * B  # the bucketed path ran
        eng.apply_gradients()
    ent_after, rel_after = (x.cpu().numpy() for x in eng.get_embeddings())
    out += [eng.read_loss(), ent_after, rel_after]
    eng.close()
    return out


def _compare(a, b, fused=True):
    if fused:
        assert (a[0] == b[0]).all() and (a[1] == b[1]).all()  # scores bit-equal
        assert abs(a[4] - b[4]) <= 1e-6 * abs(b[4])
    assert _close(a[2], b[2], 2e-5) and _close(a[3], b[3], 2e-5)
    assert _close(a[5], b[5], 1e-5) and _close(a[6], b[6], 1e-5)


@pytest.mark.parametrize("model,k,eta,E,B", [("ComplEx", 200, 10, 2000, 3000), ("HolE", 50, 7, 900, 777),
                                             ("DistMult", 400, 20, 3000, 2000),  # NIT = 4 rows (cfg3's shape)
                                             ("DistMult", 7, 3, 500, 1000), ("ComplEx", 30, 1, 300, 501), ("HolE", 13, 32, 400, 333),
                                             ("DistMult", 8, 5, 100000, 20000)])  # 13 tiles of the two-level scan
def test_bucketed_replaced_rows_equal_scatter(model, k, eta, E, B, monkeypatch):
    """Philox corruptions, three steps on one handle (the per-entity counts must reset themselves between steps)."""
    rng = np.random.default_rng(11)
    R = 9
    t = _zipf_triples(E, R, B, rng)
    a = _run("scatter", model, k, eta, E, R, t, None, monkeypatch, steps=3)
    b = _run("gather", model, k, eta, E, R, t, None, monkeypatch, steps=3)
    _compare(b, a)


def test_bucketed_replaced_rows_cfg2_full_size(monkeypatch):
    """bench.py's workload: ComplEx k=200, eta=10, 14,505 entities, 237 relations, 27,212 Zipf positives."""
    rng = np.random.default_rng(13)
    E, R, B = 14505, 237, 27212
    t = _zipf_triples(E, R, B, rng)
    a = _run("scatter", "ComplEx", 200, 10, E, R, t, None, monkeypatch, steps=2)
    b = _run("gather", "ComplEx", 200, 10, E, R, t, None, monkeypatch, steps=2)
    _compare(b, a)


@pytest.mark.parametrize("model,k,eta", [("ComplEx", 200, 10), ("DistMult", 33, 5)])
def test_bucketed_replaced_rows_skewed_injected_negatives(model, k, eta, monkeypatch):
    """Every corruption replaces one of 3 entities: buckets of thousands of entries, split over many warps."""
    rng = np.random.default_rng(17)
    E, R, B = 700, 7, 4000
    t = _zipf_triples(E, R, B, rng)
    neg = (rng.choice(np.array([3, 77, 500], np.int32), B * eta), rng.integers(0, 2, B * eta).astype(np.uint8))
    a = _run("scatter", model, k, eta, E, R, t, neg, monkeypatch, steps=2)
    b = _run("gather", model, k, eta, E, R, t, neg, monkeypatch, steps=2)
    _compare(b, a)


@pytest.mark.parametrize("model,k,eta", [("ComplEx", 200, 10), ("DistMult", 50, 6)])
def test_bucketed_replaced_rows_backward_ext(model, k, eta, monkeypatch):
    """KGE_STEP_BACKWARD_EXT: the caller's dL/dscore goes through the bucket the same way."""
    rng = np.random.default_rng(19)
    E, R, B = 1200, 11, 2500
    t = _zipf_triples(E, R, B, rng)
    neg = (rng.integers(0, E, B * eta).astype(np.int32), rng.integers(0, 2, B * eta).astype(np.uint8))
    ext = (rng.standard_normal(B).astype(np.float32), rng.standard_normal(eta * B).astype(np.float32))
    a = _run("scatter", model, k, eta, E, R, t, neg, monkeypatch, mode=_lib.STEP_BACKWARD_EXT, ext=ext)
    b = _run("gather", model, k, eta, E, R, t, neg, monkeypatch, mode=_lib.STEP_BACKWARD_EXT, ext=ext)
    _compare(b, a, fused=False)


def test_train_workspace_bytes():
    """kge_train_workspace_bytes: counts and offsets per entity, one total per scan tile, five ints/floats per corruption
    on the resident path; 0 where it does not apply (RotatE has its own kernel; fewer corruptions than entities)."""
    eng = _engine("ComplEx", 200, 10, 14505, 237)
    need = int(eng.lib.kge_train_workspace_bytes(eng.h, 27212))
    least = 4 * (2 * 14505 + 1) + 4 * 2 + 5 * 4 * 10 * 27212
    assert least <= need <= least + 8 * 16
    assert int(eng.lib.kge_train_workspace_bytes(eng.h, 1450)) == 0  # 14,500 corruptions < 14,505 entities
    eng.close()
    eng = _engine("RotatE", 50, 10, 500, 7)
    assert int(eng.lib.kge_train_workspace_bytes(eng.h, 1000)) == 0
    eng.close()
