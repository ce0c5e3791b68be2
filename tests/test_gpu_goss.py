"""GPU: GOSS on the device (lightgbm_b200/csrc/goss_kernel.cuh) against the definition of GOSSStrategy::Helper
(reference src/boosting/goss.hpp:118-167), byte for byte against tests/helpers.py goss_reference, whose draws are the
device's counter-based uniforms (tests/test_gpu_boosting_exact.py covers the edge sizes, keys and rates); and the tree
grown on the sampled set equals the oracle's tree on the same set and the same rescaled gradients."""
import numpy as np
import pytest

from helpers import compare_trees, goss_reference, synth_identity

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n,top,other", [(200_000, 0.2, 0.1), (50_001, 0.05, 0.3), (1000, 0.5, 0.5)])
def test_goss_sample_definition(built_lib, n, top, other):
    """The bag and the rescaled arrays equal the restatement byte for byte (tests/helpers.py goss_reference); the same
    iteration draws the same bag, another iteration another."""
    import lightgbm_b200 as lgb
    from lightgbm_b200.tree_learner import DeviceArray
    bins, y, g, h = synth_identity(n, 8, seed=n)
    rng = np.random.default_rng(5)
    h = (0.05 + rng.random(n)).astype(np.float32)
    L = lgb.B200TreeLearner(lgb.Config(num_leaves=15))
    L.init(lgb.Layout.identity(bins))
    dg, dh = DeviceArray(n * 4).upload(g), DeviceArray(n * 4).upload(h)
    cnt = L.goss_sample(dg, dh, top, other, seed=7, iteration=11)
    bag = L.get_bagging_data(cnt)
    want_bag, want_g, want_h = goss_reference(g, h, top, other, 7, 11)
    assert bag.tobytes() == want_bag.tobytes()
    assert dg.download(np.float32, n).tobytes() == want_g.tobytes()
    assert dh.download(np.float32, n).tobytes() == want_h.tobytes()
    dg.upload(g); dh.upload(h)
    cnt2 = L.goss_sample(dg, dh, top, other, seed=7, iteration=11)
    assert cnt2 == cnt and np.array_equal(L.get_bagging_data(cnt2), bag)
    dg.upload(g); dh.upload(h)
    cnt3 = L.goss_sample(dg, dh, top, other, seed=7, iteration=12)
    assert L.get_bagging_data(cnt3).tobytes() == goss_reference(g, h, top, other, 7, 12)[0].tobytes()


def test_tree_on_goss_sample_matches_oracle(built_lib):
    import lightgbm_b200 as lgb
    from lightgbm_b200.tree_learner import DeviceArray
    from oracle import oracle_py
    n, f = 60000, 16
    bins, y, g, h = synth_identity(n, f, seed=31)
    h = (0.2 + np.random.default_rng(2).random(n)).astype(np.float32)
    lay = lgb.Layout.identity(bins)
    L = lgb.B200TreeLearner(lgb.Config(num_leaves=31))
    L.init(lay)
    dg, dh = DeviceArray(n * 4).upload(g), DeviceArray(n * 4).upload(h)
    cnt = L.goss_sample(dg, dh, 0.2, 0.1, seed=1, iteration=20)
    bag = L.get_bagging_data(cnt)
    t = L.train(dg, dh)
    o = oracle_py.train_tree(lay, dg.download(np.float32, n), dh.download(np.float32, n), bag_indices=bag, num_leaves=31)
    matched, diverged = compare_trees(t, o, 1e-5)
    assert diverged or matched == o.num_leaves - 1
    # graph replay with a bag of a different size (no re-capture needed: the count lives on the device)
    dg.upload(g); dh.upload(h)
    cnt2 = L.goss_sample(dg, dh, 0.1, 0.05, seed=1, iteration=21)
    bag2 = L.get_bagging_data(cnt2)
    assert cnt2 != cnt
    t2 = L.train(dg, dh)
    o2 = oracle_py.train_tree(lay, dg.download(np.float32, n), dh.download(np.float32, n), bag_indices=bag2, num_leaves=31)
    matched, diverged = compare_trees(t2, o2, 1e-5)
    assert diverged or matched == o2.num_leaves - 1


def test_goss_booster_learns(built_lib):
    """data_sample_strategy=goss through the booster mirror: the loss keeps falling once sampling starts."""
    import lightgbm_b200 as lgb
    n, f = 80000, 12
    bins, y, g, h = synth_identity(n, f, seed=9)
    B = lgb.B200Booster(lgb.Layout.identity(bins), y, lgb.Config(num_leaves=31), learning_rate=0.2, data_sample_strategy="goss",
                        top_rate=0.2, other_rate=0.1)
    losses = []
    for _ in range(12):
        B.update(); losses.append(B.l2())
    assert all(b < a for a, b in zip(losses, losses[1:])), losses
