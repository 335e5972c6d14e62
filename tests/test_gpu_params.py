"""GPU, at the C ABI: how the DiT, VAE decoder and VAE encoder handles take a reference state_dict.

For a depth-1 DiT, the shipped decoder and the shipped encoder:
* every required key is required: finalize without it fails with TPX_ERR_STATE and names the key; leaving out exactly the optional
  keys (the DiT's null_cond_embedding and its cross- / self-attention biases) succeeds;
* an unknown key is TPX_ERR_KEY, a wrong rank or dimension TPX_ERR_SHAPE;
* the other half's keys (the encoder's for the decoder and the reverse) return 1 and count for nothing;
* a run before finalize, or after a later set_weight, is TPX_ERR_STATE, and a set_weight drops the DiT's timestep table;
* tpx_dit_get_weight gives back the fp16 of every key set.
"""
import ctypes as C

import pytest
import torch

from tpxl_b200 import _lib, synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
OK, ERR_ARG, ERR_SHAPE, ERR_STATE, ERR_KEY = 0, -1, -3, -4, -5

# the small configuration test_gpu_dit.py runs end to end
DIT_CFG = dict(seq_length=128, in_channels=8, condition_channels=64, hidden_size=128, depth=1, num_heads=4, attn_proj_bias=True,
               cond_drop_prob=0.1)
DIT_SHAPES = synth.dit_shapes(**DIT_CFG)
DIT_OPTIONAL = {"null_cond_embedding"} | {f"blocks.0.{m}.bias" for m in ("crossattn.to_q", "crossattn.to_k", "crossattn.to_v",
                                                                          "crossattn.proj", "attn.qkv", "attn.proj")}
DEC_SHAPES = synth.vae_decoder_shapes()
ENC_SHAPES = synth.vae_encoder_shapes()


class Kind:
    def __init__(self, name, prefix, shapes, optional, other, make_cfg, seed):
        self.name, self.prefix, self.shapes, self.optional, self.other, self.make_cfg, self.seed = name, prefix, shapes, optional, other, make_cfg, seed

    def fn(self, what):
        return getattr(_lib.lib(), f"{self.prefix}_{what}")

    def create(self):
        h = C.c_void_p()
        cfg = self.make_cfg()
        assert self.fn("create")(C.byref(cfg), C.byref(h)) == OK, _lib.lib().tpx_last_error()
        return h

    @property
    def required(self):
        return [k for k in self.shapes if k not in self.optional]


KINDS = {
    "dit": Kind("dit", "tpx_dit", DIT_SHAPES, DIT_OPTIONAL, None,
                lambda: _lib.DitConfig(128, 8, 16, 64, 128, 1, 4, 512), 31),
    "vae": Kind("vae", "tpx_vae", DEC_SHAPES, set(), ENC_SHAPES, lambda: _lib.VaeConfig(1, 6, 256, 32, 8), 32),
    "enc": Kind("enc", "tpx_vae_encoder", ENC_SHAPES, set(), DEC_SHAPES, lambda: _lib.VaeConfig(1, 6, 256, 32, 8), 33),
}
_SD = {}


def _sd(name):
    if name not in _SD:
        k = KINDS[name]
        sd = synth.synth_state_dict(k.shapes, k.seed)
        if k.other is not None:
            sd.update(synth.synth_state_dict(k.other, k.seed + 100))
        _SD[name] = {key: v.to(DEV) for key, v in sd.items()}
    return _SD[name]


def _set(kind, h, key, t, shape=None):
    shape = tuple(t.shape) if shape is None else shape
    arr = (C.c_int64 * len(shape))(*shape)
    return kind.fn("set_weight")(h, key.encode(), t.data_ptr(), _lib.DTYPE_F32, arr, len(shape), _lib.stream_ptr())


def _fill(kind, h, skip=()):
    sd = _sd(kind.name)
    for key in kind.shapes:
        if key not in skip:
            assert _set(kind, h, key, sd[key]) == OK, (key, _lib.lib().tpx_last_error())


def _finalize(kind, h):
    return kind.fn("finalize")(h, _lib.stream_ptr())


def _err():
    return _lib.lib().tpx_last_error().decode()


@pytest.fixture
def handle(request):
    kind = KINDS[request.param]
    h = kind.create()
    yield kind, h
    torch.cuda.synchronize()
    kind.fn("destroy")(h)


def _all(names=KINDS):
    return pytest.mark.parametrize("handle", list(names), indirect=True)


@pytest.mark.parametrize("handle,key", [(n, k) for n, kind in KINDS.items() for k in kind.required], indirect=["handle"])
def test_missing_required_key(handle, key):
    kind, h = handle
    _fill(kind, h, skip={key})
    assert _finalize(kind, h) == ERR_STATE
    msg = _err()
    assert f"'{key}'" in msg and "finalize" in msg, msg


@_all()
def test_optional_keys_may_be_omitted(handle):
    kind, h = handle
    _fill(kind, h, skip=kind.optional)
    assert _finalize(kind, h) == OK, _err()


@_all()
def test_unknown_key(handle):
    kind, h = handle
    t = _sd(kind.name)[kind.required[0]]
    bad = {"dit": ["blocks.1.mlp.fc1.weight", "blocks.0.mlp.fc3.weight", "blocks.x.mlp.fc1.weight", "pos_embed"],
           "vae": ["decoder.up_blocks.0.nets.0.shortcut.weight", "decoder.mid_block.nets.2.norm1.weight", "decoder.bogus"],
           "enc": ["encoder.down_blocks.0.nets.0.shortcut.weight", "encoder.mid_block.nets.2.norm1.weight", "encoder.bogus"]}[kind.name]
    for key in bad:
        assert _set(kind, h, key, t, shape=tuple(t.shape)) == ERR_KEY, key
        assert key in _err() and "set_weight" in _err()


@_all()
def test_wrong_shape(handle):
    kind, h = handle
    sd = _sd(kind.name)
    for key in kind.shapes:
        t = sd[key]
        shp = tuple(t.shape)
        assert _set(kind, h, key, t, shape=shp + (1,)) == ERR_SHAPE, key
        assert key in _err()
        if len(shp) > 1:
            assert _set(kind, h, key, t, shape=shp[:-1]) == ERR_SHAPE, key
        for d in range(len(shp)):
            wrong = shp[:d] + (shp[d] + 1,) + shp[d + 1:]
            assert _set(kind, h, key, t, shape=wrong) == ERR_SHAPE, (key, wrong)


@_all(["vae", "enc"])
def test_other_half_is_ignored(handle):
    kind, h = handle
    sd = _sd(kind.name)
    for key in kind.other:
        assert _set(kind, h, key, sd[key]) == 1, key
    assert _finalize(kind, h) == ERR_STATE
    _fill(kind, h)
    for key in kind.other:
        assert _set(kind, h, key, sd[key]) == 1, key
    assert _finalize(kind, h) == OK, _err()


def _null_argument(kind, h):
    assert kind.fn("set_weight")(h, None, 1, _lib.DTYPE_F32, (C.c_int64 * 1)(1), 1, None) == ERR_ARG
    assert kind.fn("set_weight")(None, b"x", 1, _lib.DTYPE_F32, (C.c_int64 * 1)(1), 1, None) == ERR_ARG
    assert kind.fn("finalize")(None, None) == ERR_ARG


@_all()
def test_null_arguments(handle):
    _null_argument(*handle)


@_all(["vae", "enc"])
def test_vae_run_needs_finalize(handle):
    kind, h = handle
    lib = _lib.lib()
    P = 2
    ws_bytes = kind.fn("workspace_bytes")(h, P)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)
    if kind.name == "vae":
        x = torch.randn(P, 1, 4, 4, 4, device=DEV)
        out = torch.empty(P, 6, 8, 8, 8, device=DEV)
        run = lambda: lib.tpx_vae_decode(h, x.data_ptr(), _lib.DTYPE_F32, out.data_ptr(), _lib.DTYPE_F32, P, ws.data_ptr(), ws_bytes, _lib.stream_ptr())
    else:
        x = torch.randn(P, 6, 8, 8, 8, device=DEV)
        out = torch.empty(P, 2, 4, 4, 4, device=DEV)
        run = lambda: lib.tpx_vae_encode(h, x.data_ptr(), _lib.DTYPE_F32, out.data_ptr(), _lib.DTYPE_F32, P, ws.data_ptr(), ws_bytes, _lib.stream_ptr())
    assert run() == ERR_STATE
    _fill(kind, h)
    assert run() == ERR_STATE
    assert _finalize(kind, h) == OK, _err()
    assert run() == OK, _err()
    key = kind.required[-1]
    assert _set(kind, h, key, _sd(kind.name)[key]) == OK
    assert run() == ERR_STATE
    assert _finalize(kind, h) == OK
    assert run() == OK, _err()
    torch.cuda.synchronize()


def _dit_buffers(lib, h, n_seq):
    N, Cin, Dc, M = 128, 8, 64, 4
    x = torch.randn(1, N, Cin, device=DEV)
    y = torch.randn(1, M, Dc, device=DEV)
    out = torch.empty(1, N, 16, dtype=torch.float16, device=DEV)
    cb = lib.tpx_dit_cond_bytes(h, 1, M)
    cond = torch.empty(cb, dtype=torch.uint8, device=DEV)
    wb = lib.tpx_dit_workspace_bytes(h, n_seq)
    ws = torch.empty(wb, dtype=torch.uint8, device=DEV)
    return x, y, M, out, cond, cb, ws, wb


@_all(["dit"])
def test_dit_run_needs_finalize(handle):
    kind, h = handle
    lib, st = _lib.lib(), _lib.stream_ptr()
    x, y, M, out, cond, cb, ws, wb = _dit_buffers(lib, h, 1)
    t = torch.tensor([500], dtype=torch.int64, device=DEV)
    set_cond = lambda: lib.tpx_dit_set_cond(h, y.data_ptr(), 1, M, cond.data_ptr(), cb, st)
    fwd = lambda: lib.tpx_dit_forward(h, x.data_ptr(), t.data_ptr(), 1, 0, 1.0, out.data_ptr(), ws.data_ptr(), wb, st)
    assert set_cond() == ERR_STATE
    assert fwd() == ERR_STATE
    _fill(kind, h)
    assert set_cond() == ERR_STATE
    assert _finalize(kind, h) == OK, _err()
    assert set_cond() == OK, _err()
    assert fwd() == OK, _err()
    assert _set(kind, h, "x_embedder.bias", _sd("dit")["x_embedder.bias"]) == OK
    assert fwd() == ERR_STATE
    assert set_cond() == ERR_STATE
    assert _finalize(kind, h) == OK
    assert set_cond() == OK and fwd() == OK, _err()
    torch.cuda.synchronize()


@_all(["dit"])
def test_dit_set_weight_drops_timestep_table(handle):
    kind, h = handle
    lib, st = _lib.lib(), _lib.stream_ptr()
    x, y, M, out, cond, cb, ws, wb = _dit_buffers(lib, h, 1)
    _fill(kind, h)
    assert _finalize(kind, h) == OK, _err()
    assert lib.tpx_dit_set_cond(h, y.data_ptr(), 1, M, cond.data_ptr(), cb, st) == OK
    ts = (C.c_int64 * 2)(999, 500)
    tb = lib.tpx_dit_timesteps_bytes(h, 2)
    table = torch.empty(tb, dtype=torch.uint8, device=DEV)
    assert lib.tpx_dit_set_timesteps(h, ts, 2, table.data_ptr(), tb, st) == OK, _err()
    step = lambda: lib.tpx_dit_forward_step(h, x.data_ptr(), 500, 1, 0, 1.0, out.data_ptr(), ws.data_ptr(), wb, st)
    assert step() == OK, _err()
    assert _set(kind, h, "t_embedder.mlp.0.bias", _sd("dit")["t_embedder.mlp.0.bias"]) == OK
    assert _finalize(kind, h) == OK
    assert lib.tpx_dit_set_cond(h, y.data_ptr(), 1, M, cond.data_ptr(), cb, st) == OK
    assert step() == ERR_STATE
    assert "timestep" in _err()
    torch.cuda.synchronize()


@_all(["dit"])
def test_dit_get_weight_returns_fp16(handle):
    kind, h = handle
    lib, st = _lib.lib(), _lib.stream_ptr()
    sd = _sd("dit")
    _fill(kind, h)
    assert _finalize(kind, h) == OK, _err()
    for key, t in sd.items():
        got = torch.full_like(t, float("nan"), dtype=torch.float16)
        assert lib.tpx_dit_get_weight(h, key.encode(), got.data_ptr(), _lib.DTYPE_F16, st) == OK, key
        torch.cuda.synchronize()
        assert torch.equal(got, t.half()), key
    assert lib.tpx_dit_get_weight(h, b"blocks.1.mlp.fc1.weight", got.data_ptr(), _lib.DTYPE_F16, st) == ERR_KEY
