"""RealESRNet x4 kernels against float64 at the production shape: 16 faces of 256 x 256 -> 1024 x 1024 (the face swap's
step 2).  Every convolution shape and epilogue of RRDBNet on its own fp32 inputs, then the whole forward and process().
The float64 references are plain torch on the GPU.  Tolerances are the measured errors (H100 80GB HBM3) with headroom;
each test prints what it measured."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import REL_TOL, rel_err, rel_rms
from oracle import sr_oracle as SO

pytestmark = pytest.mark.gpu

B, SIZE = 16, 256
CONV_TOL = 5e-5


def _check(ours, ref64, tol, what):
    e, r = rel_err(ours, ref64), rel_rms(ours, ref64)
    print(f"{what}: max-rel {e:.2e}  rel-RMS {r:.2e}")
    assert e <= tol and r <= tol, (what, e, r)
    return e


@pytest.fixture(autouse=True)
def _no_grad():
    """Every test runs without autograd (the network is forward-only); the setting is restored after it."""
    with torch.no_grad():
        yield


@pytest.fixture(scope="module")
def net():
    from e4s_b200.gpen.sr_model.rrdbnet_arch import RRDBNet
    m = RRDBNet(num_in_ch=3, num_out_ch=3, num_feat=32, num_block=23, num_grow_ch=32, scale=4)
    m.load_state_dict(SO.synthetic_state(), strict=True)
    return m.eval().requires_grad_(False).cuda()


@pytest.fixture(scope="module")
def images():
    u8 = np.stack([SO.case_image(SIZE, SIZE, 100 + i) for i in range(B)])
    return torch.from_numpy(u8[..., ::-1].copy()).permute(0, 3, 1, 2).cuda().float() / 255    # RGB, as process() feeds it


@pytest.fixture(scope="module")
def st64():
    return {k: v.double().cuda() for k, v in SO.synthetic_state().items()}


def _randn(*shape, seed, dev="cuda"):
    return torch.randn(*shape, generator=torch.Generator(device=dev).manual_seed(seed), device=dev)


def _weights(cout, cin, seed):
    from e4s_b200.encoders.psp_encoders import _conv_planes
    w = _randn(cout, cin, 3, 3, seed=seed, dev="cpu") * (2.0 / (9 * cin)) ** 0.5
    b = 0.1 * _randn(cout, seed=seed + 1)
    return w, _conv_planes(w).cuda(), b


def _ref(x_pm, w, b, up=False):
    x = x_pm.permute(0, 3, 1, 2).double()
    if up:
        x = F.interpolate(x, scale_factor=2, mode="nearest")
    return (F.conv2d(x, w.double().cuda(), padding=1) + b.double()[None, :, None, None]).permute(0, 2, 3, 1)


def _lrelu(t):
    return torch.where(t > 0, t, 0.2 * t)


@pytest.fixture(scope="module")
def dense_buffer():
    """A residual dense block's [B, 256, 256, 160] buffer: x, x1 .. x4 at channel offsets 0, 32, .., 128."""
    return _lrelu(_randn(B, SIZE, SIZE, 160, seed=7))


@pytest.mark.parametrize("k", [1, 2, 3, 4])
def test_rdb_conv_into_its_buffer(dense_buffer, k):
    """conv k of a residual dense block: channels [0, 32k) of the buffer in, 32 channels at offset 32k of the same buffer
    out, leaky ReLU 0.2 (channels outside the written slice are untouched)."""
    from e4s_b200 import kernels as K
    buf = dense_buffer.clone()
    w, planes, b = _weights(32, 32 * k, seed=10 + k)
    ref = _lrelu(_ref(buf[..., :32 * k], w, b))
    out = K.conv3x3_dense_tc(buf[..., :32 * k], planes, b, out=buf[..., 32 * k:32 * k + 32], lrelu=0.2)
    assert out.data_ptr() == buf.data_ptr() + 4 * 32 * k
    _check(buf[..., 32 * k:32 * k + 32], ref, CONV_TOL, f"rdb conv{k} {32 * k}->32 lrelu")
    assert torch.equal(buf[..., :32 * k], dense_buffer[..., :32 * k]) and torch.equal(buf[..., 32 * k + 32:],
                                                                                      dense_buffer[..., 32 * k + 32:])


@pytest.mark.parametrize("residuals", [1, 2])
def test_rdb_conv5(dense_buffer, residuals):
    """conv5: x5 * 0.2 + x into channel 0 of the next block's buffer; with two residuals also the RRDB's (.) * 0.2 + x,
    where x is read from the very elements the result overwrites (a block's first buffer)."""
    from e4s_b200 import kernels as K
    w, planes, b = _weights(32, 160, seed=20)
    nxt = _randn(B, SIZE, SIZE, 160, seed=21)
    x_blk = nxt[..., :32].double()
    t = _ref(dense_buffer, w, b) * 0.2 + dense_buffer[..., :32].double()
    if residuals == 1:
        K.conv3x3_dense_tc(dense_buffer, planes, b, out=nxt[..., :32], alpha=0.2, r0=dense_buffer[..., :32])
    else:
        t = t * 0.2 + x_blk
        K.conv3x3_dense_tc(dense_buffer, planes, b, out=nxt[..., :32], alpha=0.2, r0=dense_buffer[..., :32], beta=0.2,
                           r1=nxt[..., :32])
    _check(nxt[..., :32], t, CONV_TOL, f"rdb conv5 160->32, {residuals} residual(s)")


def test_conv_body_and_trunk_residual(dense_buffer):
    from e4s_b200 import kernels as K
    w, planes, b = _weights(32, 32, seed=30)
    out = torch.empty_like(dense_buffer)
    feat = _randn(B, SIZE, SIZE, 160, seed=31)
    K.conv3x3_dense_tc(dense_buffer[..., :32], planes, b, out=out[..., :32], r0=feat[..., :32])
    _check(out[..., :32], _ref(dense_buffer[..., :32], w, b) + feat[..., :32].double(), CONV_TOL, "conv_body + feat")


@pytest.mark.parametrize("side,pitch", [(SIZE, 160), (2 * SIZE, 32)])
def test_up_conv_fused_nearest(side, pitch):
    """conv_up1 (256 -> 512, reading a channel slice of a 160-channel buffer) and conv_up2 (512 -> 1024): nearest 2x
    up-sampling in the halo copy, leaky ReLU."""
    from e4s_b200 import kernels as K
    src = _randn(B, side, side, pitch, seed=side)
    w, planes, b = _weights(32, 32, seed=40 + pitch)
    out = K.conv3x3_dense_tc(src[..., :32], planes, b, up=True, lrelu=0.2)
    assert tuple(out.shape) == (B, 2 * side, 2 * side, 32)
    _check(out, _lrelu(_ref(src[..., :32], w, b, up=True)), CONV_TOL, f"conv_up {side}->{2 * side}")


def test_conv_hr():
    from e4s_b200 import kernels as K
    x = _lrelu(_randn(B, 4 * SIZE, 4 * SIZE, 32, seed=50))
    w, planes, b = _weights(32, 32, seed=51)
    _check(K.conv3x3_dense_tc(x, planes, b, lrelu=0.2), _lrelu(_ref(x, w, b)), CONV_TOL, "conv_hr 1024^2")


def test_conv_first_and_last():
    from e4s_b200 import kernels as K
    img = torch.rand(B, 3, SIZE, SIZE, device="cuda")
    w, _, b = _weights(32, 3, seed=60)
    buf = torch.zeros(B, SIZE, SIZE, 160, device="cuda")
    K.conv3x3_rgb(img, w.cuda(), b, out=buf[..., :32])
    ref = F.conv2d(img.double(), w.double().cuda(), b.double(), padding=1)
    _check(buf[..., :32], ref.permute(0, 2, 3, 1), 1e-5, "conv_first 3->32")
    assert int(torch.count_nonzero(buf[..., 32:])) == 0
    x = _lrelu(_randn(B, 4 * SIZE, 4 * SIZE, 32, seed=61))
    w, _, b = _weights(3, 32, seed=62)
    ours = K.conv3x3_rgb(x, w.cuda(), b)
    _check(ours, F.conv2d(x.permute(0, 3, 1, 2).double(), w.double().cuda(), b.double(), padding=1), 1e-5, "conv_last 32->3")


@pytest.mark.parametrize("cin", [32, 160])
def test_resident_and_streaming_weights_bitwise(monkeypatch, dense_buffer, cin):
    from e4s_b200 import kernels as K
    _, planes, b = _weights(32, cin, seed=70)
    resident = K.conv3x3_dense_tc(dense_buffer[..., :cin], planes, b, lrelu=0.2)
    monkeypatch.setenv("E4S_B200_RS_STREAM", "1")
    streamed = K.conv3x3_dense_tc(dense_buffer[..., :cin], planes, b, lrelu=0.2)
    assert torch.equal(resident, streamed)


def test_dense_entry_rejects_bad_operands(dense_buffer):
    from e4s_b200 import _lib
    from e4s_b200 import kernels as K
    _, planes, b = _weights(32, 64, seed=80)
    with pytest.raises(RuntimeError):                                 # overlapping pitch: not a slice of a buffer
        K.conv3x3_dense_tc(dense_buffer[..., :64].transpose(1, 2), planes, b)
    lib, x, y = _lib.load(), dense_buffer, torch.empty(1, 8, 8, 32, device="cuda")
    call = lambda x_ld, y_ld, xp=x.data_ptr(): lib.e4s_conv3x3_dense_tcr_f32(  # noqa: E731
        xp, x_ld, planes.data_ptr(), b.data_ptr(), 1.0, None, 1.0, None, y.data_ptr(), y_ld, 1, 8, 8, 64, 32, 0, 1.0, None)
    assert call(48, 32) == -1                                         # pitch below the channel count
    assert call(160, 30) == -1
    assert call(162, 32) == -3                                        # pitch not a multiple of 4
    assert call(160, 32, x.data_ptr() + 8) == -3                      # operand not 16-byte aligned
    assert call(160, 32) == 0
    torch.cuda.synchronize()


@pytest.fixture(scope="module")
def forward_pair(net, images, st64):
    ours = net(images)
    ref = SO.rrdbnet_forward(st64, images.double())
    return ours, ref


def test_forward_against_float64(forward_pair):
    ours, ref = forward_pair
    assert tuple(ours.shape) == (B, 3, 4 * SIZE, 4 * SIZE)
    _check(ours, ref, REL_TOL, "RRDBNet.forward 16 x 256^2 -> 1024^2")
    print(f"max abs error {float((ours.double() - ref).abs().max()):.2e}, image std {float(ref.std()):.3f}")


def test_alone_equals_batch_and_graph_replay(net, images, forward_pair):
    full = forward_pair[0]
    alone = net(images[5:6].contiguous())
    assert torch.equal(alone[0], full[5])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        net(images[:4])
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    x = images[:4].clone()
    with torch.cuda.graph(g):
        out = net(x)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, full[:4])


def test_process_bytes_against_float64(tmp_path, st64):
    """process() on a 256 x 256 uint8 BGR face: equal to the float64 bytes except where the float64 value lies within twice
    the measured error of a rounding boundary, and never more than 1 off."""
    from e4s_b200.gpen.sr_model.real_esrnet import RealESRNet
    os.makedirs(tmp_path / "weights")
    torch.save({"params_ema": SO.synthetic_state()}, tmp_path / "weights" / "realesrnet_x4.pth")
    sr = RealESRNet(str(tmp_path), "realesrnet", 4, device="cuda")
    img = SO.case_image(SIZE, SIZE, 200)
    ours = sr.process(img)
    assert ours.dtype == np.uint8 and ours.shape == (4 * SIZE, 4 * SIZE, 3)
    x = SO.to_input(img).cuda()
    out32 = sr.srmodel(x)[0]
    ref = SO.rrdbnet_forward(st64, x.double())[0]
    E = float((out32.double() - ref).abs().max())
    v = (ref.clamp(0, 1) * 255).permute(1, 2, 0)[:, :, [2, 1, 0]].cpu().numpy()
    ref_u8 = np.round(v).astype(np.int64)
    diff = np.abs(ours.astype(np.int64) - ref_u8)
    near = np.abs(v - np.floor(v) - 0.5) <= 2 * E * 255
    print(f"process: E = {E:.2e}, bytes off by 1: {int((diff == 1).sum())}, near a boundary: {int(near.sum())} of {v.size}")
    assert diff.max() <= 1 and not (diff[~near]).any()


def test_ragged_size_against_float64(net, st64):
    x = torch.rand(2, 3, 100, 76, device="cuda")
    _check(net(x), SO.rrdbnet_forward(st64, x.double()), REL_TOL, "RRDBNet.forward 2 x 100x76")


def test_forward_rejects_bad_inputs(net):
    with pytest.raises(ValueError):
        net(torch.zeros(1, 3, 16, 16))                                 # CPU tensor
    with pytest.raises(ValueError):
        net(torch.zeros(1, 3, 16, 16, device="cuda", dtype=torch.float16))
    with pytest.raises(ValueError):
        net(torch.zeros(1, 4, 16, 16, device="cuda"))
    from e4s_b200.gpen.sr_model.rrdbnet_arch import RRDBNet
    with pytest.raises(NotImplementedError):
        RRDBNet(3, 3, scale=2, num_feat=32, num_block=1, num_grow_ch=32).cuda()(torch.zeros(1, 3, 16, 16, device="cuda"))
