"""CPU: the compact training input (DESIGN.md §18).  The argument checks of forward_train's uint8 path, of the uint8
stem and of the losses' vertex_weights=None; the layout the uint8 stem pack writes (S and convraw.0's image and pad
channels), restated in numpy; and the weights the losses take from the mask, against the loader's
mask.unsqueeze(0).float()."""
import numpy as np
import pytest
import torch

from oracle import loss_oracle as lo
from pvnet_b200 import conv as pc
from pvnet_b200 import net_utils as nu
from pvnet_b200.model_repository import Resnet18_8s
from tests.train_u8_oracle import IMAGENET_MEAN, IMAGENET_STD, mask_weights, normalise, pack_u8

F32 = np.float32


def _image(b, H, W, seed=0):
    return np.random.default_rng(seed).integers(0, 256, (b, H, W, 3), dtype=np.uint8)


# ----------------------------------------------------------------------------- the pack's oracle
def test_normalise_is_torchvision_to_tensor_and_normalize_on_the_cpu():
    img = _image(2, 6, 10)
    want = torch.from_numpy(img).permute(0, 3, 1, 2).float().div(255)          # ToTensor
    mean = torch.tensor(IMAGENET_MEAN).view(1, 3, 1, 1)
    std = torch.tensor(IMAGENET_STD).view(1, 3, 1, 1)
    want = want.sub(mean).div(std)                                               # Normalize
    assert normalise(img, IMAGENET_MEAN, IMAGENET_STD).tobytes() == want.numpy().tobytes()
    # every byte value in every channel: the sequence is three correctly rounded fp32 ops
    allv = np.arange(256, dtype=np.uint8).reshape(1, 16, 16, 1).repeat(3, 3)
    got = normalise(allv, IMAGENET_MEAN, IMAGENET_STD)
    for c in range(3):
        v = (np.arange(256, dtype=F32) / F32(255) - F32(IMAGENET_MEAN[c])) / F32(IMAGENET_STD[c])
        assert got[0, c].reshape(-1).tobytes() == v.tobytes()


@pytest.mark.parametrize("cs,co", [(40, 32), (8, 0), (48, 36)])
def test_pack_layout(cs, co):
    b, H, W = 2, 6, 10
    img = _image(b, H, W, seed=cs)
    x = normalise(img, IMAGENET_MEAN, IMAGENET_STD)                            # [b,3,H,W]
    sentinel = np.full((b, H, W, cs), np.nan, F32)
    S, buf = pack_u8(img, IMAGENET_MEAN, IMAGENET_STD, sentinel.copy(), co)
    xr = pc.round_tf32(torch.from_numpy(x)).numpy()
    assert S.shape == (b, H // 2, W // 2, 16) and S.dtype == F32
    for py in range(2):
        for px in range(2):
            for c in range(3):
                assert S[..., (py * 2 + px) * 3 + c].tobytes() == \
                    np.ascontiguousarray(xr[:, c, py::2, px::2]).tobytes()
    assert (S[..., 12:] == 0).all() and not np.signbit(S[..., 12:]).any()
    # the image slice: the normalised values unrounded (the float path's cat copies the fp32 image), then 5 zeros
    assert buf[..., co:co + 3].tobytes() == np.ascontiguousarray(x.transpose(0, 2, 3, 1)).tobytes()
    assert (buf[..., co + 3:co + 8] == 0).all() and not np.signbit(buf[..., co + 3:co + 8]).any()
    rest = np.concatenate([buf[..., :co], buf[..., co + 8:]], -1)
    assert np.isnan(rest).all()                                                   # the other channels untouched


# ----------------------------------------------------------------------------- weights from the mask
@pytest.mark.parametrize("dtype", [torch.int64, torch.int32, torch.uint8, torch.bool])
def test_mask_weights_are_the_loaders(dtype):
    rng = np.random.default_rng(3)
    m = rng.integers(0, 3, (2, 5, 7))
    if dtype != torch.bool:
        m[0, 0, :3] = [2, 255, 1]
    if dtype == torch.int64:
        m[1, 0, :2] = [(1 << 24) + 1, -(1 << 40) - 3]                             # rounded to nearest by .float()
    mask = torch.from_numpy(m).to(dtype) if dtype != torch.bool else torch.from_numpy(m > 0)
    want = torch.stack([mi.unsqueeze(0).float() for mi in mask])                  # linemod_dataset.py:227, collated
    assert torch.equal(nu.mask_weights(mask), want)
    assert mask_weights(mask.numpy()).tobytes() == want.numpy().tobytes()


@pytest.mark.parametrize("dtype", [torch.int64, torch.int32, torch.uint8, torch.bool])
def test_oracle_losses_with_mask_weights(dtype):
    rng = np.random.default_rng(5)
    b, vd, h, w = 2, 6, 9, 11
    m = rng.integers(0, 2, (b, h, w))
    if dtype != torch.bool:
        m[0, 1, :4] = 2                                                           # a mask value 2 weighs 2
    mask = torch.from_numpy(m).to(dtype) if dtype != torch.bool else torch.from_numpy(m > 0)
    pred = rng.standard_normal((b, vd, h, w)).astype(F32)
    tgt = rng.standard_normal((b, vd, h, w)).astype(F32)
    want = mask.unsqueeze(1).float().numpy()
    got = mask_weights(mask.numpy())
    assert lo.smooth_l1_normalized(pred, tgt, got).tobytes() == lo.smooth_l1_normalized(pred, tgt, want).tobytes()
    assert lo.smooth_l1_elementwise(pred, tgt, got).tobytes() == lo.smooth_l1_elementwise(pred, tgt, want).tobytes()


def test_grad_mode_losses_with_none_weights_equal_the_mask_weights():
    # in grad mode the functions evaluate torch expressions (on the CPU here): None takes the weights from the mask
    g = torch.Generator().manual_seed(0)
    b, h, w, K = 2, 8, 12, 3
    seg = torch.randn(b, 3, h, w, generator=g)                                   # three classes: a value 2 is valid
    ver = torch.randn(b, 2 * K, h, w, generator=g)
    mask = torch.randint(0, 2, (b, h, w), generator=g)
    mask[0, 0, :3] = 2
    field = torch.randn(b, 2 * K, h, w, generator=g)
    for s_req in (True, False):
        a = nu.seg_vertex_losses(seg.clone().requires_grad_(s_req), ver.clone().requires_grad_(), mask, field, None)
        bb = nu.seg_vertex_losses(seg.clone().requires_grad_(s_req), ver.clone().requires_grad_(), mask, field,
                                  mask.unsqueeze(1).float())
        for u, v in zip(a, bb):
            assert torch.equal(u, v)


# ----------------------------------------------------------------------------- argument checks
def test_loss_argument_checks():
    pred = torch.zeros(2, 4, 5, 6)
    with pytest.raises(ValueError, match="vertex_weights"):
        nu.smooth_l1_loss(pred, pred, None)                                        # no mask to take them from
    seg, mask = torch.zeros(2, 2, 5, 6), torch.zeros(2, 5, 6, dtype=torch.int64)
    with pytest.raises(ValueError, match=r"\[b,1,h,w\]"):
        nu.seg_vertex_losses(seg, pred, mask, pred, torch.zeros(2, 2, 5, 6))
    with pytest.raises(ValueError, match="float32"):
        nu.seg_vertex_training_losses_from_keypoints(seg, pred, mask, torch.zeros(2, 2, 3),
                                                     torch.zeros(2, 1, 5, 6, dtype=torch.float64))
    with pytest.raises(RuntimeError, match="CUDA"):                                # None accepted, then the device
        nu.seg_vertex_training_losses(seg, pred, mask, pred, None)
    with pytest.raises(RuntimeError, match="CUDA"):
        nu.seg_vertex_training_losses_from_keypoints(seg, pred, mask, torch.zeros(2, 2, 3))
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA"):
        nu.seg_vertex_losses_from_keypoints(seg, pred, mask, torch.zeros(2, 2, 3))


def test_forward_train_argument_checks():
    net = Resnet18_8s(ver_dim=18, seg_dim=2).train()
    u8 = torch.zeros(1, 64, 64, 3, dtype=torch.uint8)
    with pytest.raises(ValueError, match="mean"):
        net.forward_train(u8)
    with pytest.raises(ValueError, match="mean"):
        net.forward_train(u8, mean=IMAGENET_MEAN)
    with pytest.raises(ValueError, match=r"\[b,H,W,3\]"):
        net.forward_train(u8.permute(0, 3, 1, 2), mean=IMAGENET_MEAN, std=IMAGENET_STD)
    with pytest.raises(ValueError, match="float image"):
        net.forward_train(torch.zeros(1, 3, 64, 64), mean=IMAGENET_MEAN, std=IMAGENET_STD)
    with pytest.raises(ValueError, match="float image"):
        net.forward_train(torch.zeros(1, 3, 64, 64), std=IMAGENET_STD)
    with pytest.raises(RuntimeError, match="CUDA"):                                # valid arguments: no CPU path
        net.forward_train(u8, mean=IMAGENET_MEAN, std=IMAGENET_STD)
    with pytest.raises(RuntimeError, match="CUDA"):
        net.forward_train(torch.zeros(1, 3, 64, 64))


def test_norm3_stem_and_upsample_argument_checks():
    w = torch.zeros(64, 3, 7, 7)
    buf = torch.zeros(1, 40, 8, 8).contiguous(memory_format=torch.channels_last)
    with pytest.raises(ValueError, match="3 values"):
        pc.norm3([0.5, 0.5], IMAGENET_STD)
    with pytest.raises(ValueError, match="3 values"):
        pc.norm3(IMAGENET_MEAN, torch.ones(4))
    m, s = pc.norm3(torch.tensor(IMAGENET_MEAN), IMAGENET_STD)
    assert list(m) == [float(F32(v)) for v in IMAGENET_MEAN] and list(s) == [float(F32(v)) for v in IMAGENET_STD]
    with pytest.raises(ValueError, match="CUDA"):
        pc.stem_train(torch.zeros(1, 8, 8, 3, dtype=torch.uint8), w, buf, 32, IMAGENET_MEAN, IMAGENET_STD)
    with pytest.raises(ValueError, match="CUDA"):
        pc.upsample2x_into(torch.zeros(1, 32, 4, 4), buf)
