"""Model inventory, checkpoint layout and round trip (SURVEY §2.4 table, §5.4)."""
import os

import pytest
import torch

from distributedmnist_b200.checkpoint import (Saver, get_checkpoint_state, resolve_checkpoint_path,
                                              step_from_path)
from distributedmnist_b200.models import dropout_keep_mask, get_model, lenet_forward, loss_and_accuracy


def test_lenet_inventory_matches_reference():
    spec, _ = get_model("lenet")
    assert spec.num_trainable == 1663370
    want = [("Variable", (5, 5, 1, 32)), ("Variable_1", (32,)), ("Variable_2", (5, 5, 32, 64)),
            ("Variable_3", (64,)), ("Variable_4", (3136, 512)), ("Variable_5", (512,)),
            ("Variable_6", (512, 10)), ("Variable_7", (10,))]
    assert [(p.ckpt_name, tuple(p.shape)) for p in spec.params] == want
    assert all(p.offset % 64 == 0 for p in spec.params) and spec.arena_numel % 2048 == 0


def test_init_distributions_and_determinism():
    spec, _ = get_model("lenet")
    a, b = spec.init_flat(66478), spec.init_flat(66478)
    assert torch.equal(a, b)
    v = spec.views(a)
    assert float(v["conv1_biases"].abs().max()) == 0.0
    assert torch.allclose(v["conv2_biases"], torch.full((64,), 0.1))
    w = v["fc1_weights"]
    assert float(w.abs().max()) <= 0.2 + 1e-6            # truncated at 2 sigma
    assert 0.08 < float(w.std()) < 0.095                  # truncated normal std = 0.88 * 0.1
    assert float(a[~spec.valid_mask()].abs().max()) == 0.0  # padding stays zero


def test_forward_shapes_loss_and_grad():
    spec, fwd = get_model("lenet")
    flat = spec.init_flat(1).requires_grad_(True)
    x = torch.randn(4, 28, 28, 1) * 0.3
    y = torch.tensor([1, 2, 3, 4])
    mask = dropout_keep_mask(123, 4, 512, 0.5)
    logits = fwd(spec.views(flat), x, train=True, keep_mask=mask)
    assert logits.shape == (4, 10)
    loss, acc = loss_and_accuracy(logits, y)
    loss.backward()
    assert flat.grad.shape == flat.shape and float(flat.grad.abs().sum()) > 0
    assert 0.0 <= float(acc) <= 1.0
    # eval mode needs no mask and is deterministic
    l1 = lenet_forward(spec.views(flat.detach()), x, train=False)
    l2 = lenet_forward(spec.views(flat.detach()), x, train=False)
    assert torch.equal(l1, l2)


def test_dropout_mask_rate_and_determinism():
    m = dropout_keep_mask(0xDEADBEEF, 256, 512, 0.5)
    assert m.shape == (256, 512) and abs(float(m.float().mean()) - 0.5) < 0.01
    assert torch.equal(m, dropout_keep_mask(0xDEADBEEF, 256, 512, 0.5))
    assert not torch.equal(m, dropout_keep_mask(0xDEADBEF0, 256, 512, 0.5))


def test_dropout_threshold_is_the_kernels():
    """The kernels compute (uint32_t)(keep_prob * 16777216.f) from an fp32 keep_prob; fp32 rounds 0.3, 0.8 and 0.99 up,
    one unit above floor(keep_prob * 2^24)."""
    import numpy as np
    from distributedmnist_b200.models.lenet import dropout_threshold
    from distributedmnist_b200.ops.selfcheck import _unhash
    sweep = [k / 100 for k in range(101)] + [0.25, 0.3, 0.75, 0.8, 0.99, 1 / 3, 0.9999999, 1e-7]
    for kp in sweep:
        device = int(np.uint32(np.float32(kp) * np.float32(16777216.0)))
        assert dropout_threshold(kp) == device, kp
    assert [dropout_threshold(k) for k in (0.3, 0.8, 0.99)] == [5033165, 13421773, 16609444]


def test_dropout_mask_decides_at_the_kernels_threshold():
    """An element whose hash lands one below the kernel's threshold is kept (floor(0.8 * 2^24) would drop it), one
    that lands on it is dropped."""
    import numpy as np
    from distributedmnist_b200.ops.selfcheck import _unhash
    for kp in (0.3, 0.8, 0.99):
        t = int(np.uint32(np.float32(kp) * np.float32(16777216.0)))
        for v, kept in ((t - 1, True), (t, False)):
            mix = _unhash((v << 8) | 0xA5)           # element 0: hash_mix(mix, 0) = fmix32(mix)
            assert bool(dropout_keep_mask(mix, 1, 1, kp)[0, 0]) == kept, (kp, v)


def test_mlp_engine_refuses_a_hidden_width_its_output_kernel_cannot_hold():
    from distributedmnist_b200.engine_cuda import CudaMlpEngine
    with pytest.raises(ValueError, match="--mlp_hidden=5184"):
        CudaMlpEngine("mlp3", 8, None, hidden=5184)


@pytest.mark.parametrize("name", ["mlp2", "mlp3"])
def test_mlp_specs(name):
    spec, fwd = get_model(name, mlp_hidden=64)
    flat = spec.init_flat(2)
    out = fwd(spec.views(flat), torch.randn(3, 28, 28, 1))
    assert out.shape == (3, 10)
    assert spec.ckpt_names()[0] == "Variable" and spec.ckpt_names()[1] == "Variable_1"


def test_checkpoint_roundtrip_and_layout(tmp_path):
    spec, _ = get_model("lenet")
    flat = spec.init_flat(3)
    saver = Saver(max_to_keep=2)
    d = str(tmp_path / "train_dir")
    for step in (10, 20, 30):
        prefix = saver.save(d, spec.to_state_dict(flat + step), step)
    assert os.path.basename(prefix) == "model.ckpt-30" and step_from_path(prefix) == 30
    st = get_checkpoint_state(d)
    assert st.model_checkpoint_path == "model.ckpt-30"
    assert st.all_model_checkpoint_paths == ["model.ckpt-20", "model.ckpt-30"]     # max_to_keep
    assert not os.path.exists(os.path.join(d, "model.ckpt-10.index"))
    text = open(os.path.join(d, "checkpoint")).read()
    assert text.startswith('model_checkpoint_path: "model.ckpt-30"')
    state, gstep = Saver.restore(resolve_checkpoint_path(d, st))
    assert gstep == 30 and set(state) == set(spec.ckpt_names())
    back = spec.from_state_dict(state)
    assert torch.equal(back[spec.valid_mask()], (flat + 30)[spec.valid_mask()])
    assert Saver.latest(d).endswith("model.ckpt-30")
    assert Saver.latest(str(tmp_path / "nope")) is None


def test_checkpoint_shape_mismatch_rejected(tmp_path):
    spec, _ = get_model("lenet")
    other, _ = get_model("mlp2", 32)
    Saver().save(str(tmp_path), other.to_state_dict(other.init_flat(0)), 1)
    state, _ = Saver.restore(Saver.latest(str(tmp_path)))
    with pytest.raises((ValueError, KeyError)):
        spec.from_state_dict(state)


def test_packed_batches_round_trip_through_the_engine_api():
    """pack_batch / load_packed (one buffer, one copy per step) feed the engine the same batch as load_batch."""
    import torch

    from distributedmnist_b200.engine import TorchEngine
    eng = TorchEngine("lenet", 8, torch.device("cpu"), lambda n: torch.zeros(n))
    g = torch.Generator().manual_seed(3)
    x, y = torch.rand(8, 28, 28, 1, generator=g) - 0.5, torch.randint(0, 10, (8,), generator=g)
    eng.load_batch(x, y)
    eng.forward_backward(0)
    ref_loss, ref_grads = eng.loss_acc()[0], eng.grads.clone()
    packed = eng.pack_batch(x, y, pin=False)
    assert packed.dtype == torch.uint8 and packed.numel() == 8 * 784 * 4 + 8 * 8
    eng.grads.zero_()
    eng.load_packed(packed)
    eng.forward_backward(0)
    assert abs(eng.loss_acc()[0] - ref_loss) < 1e-7 and torch.equal(eng.grads, ref_grads)
