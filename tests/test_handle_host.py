"""CPU: the host-side pieces the DiT, VAE and DINOv2 modules share (3dtopia-xl_b200/_lib.py) — the state-dict check and its message
on each module's shape table, the C-handle owner driven by Python stand-ins for create / destroy, and the only-growing scratch
buffer on CPU tensors.  Needs neither a GPU nor the library."""
import contextlib
import ctypes
import gc

import pytest
import torch

import tpxl_b200
from tpxl_b200 import _lib, synth
from tpxl_b200.dinov2 import Dinov2Wrapper

TINY_DIT = dict(seq_length=8, in_channels=8, condition_channels=16, hidden_size=128, depth=1, num_heads=4, attn_proj_bias=True,
                cond_drop_prob=0.1)


def _meta(shapes):
    """A state dict of the table's shapes that allocates nothing (the checks read only .shape)."""
    return {k: torch.empty(s, device="meta") for k, s in shapes.items()}


def _raises(module, sd, strict=True):
    with pytest.raises(RuntimeError) as e:
        module.load_state_dict(sd, strict=strict)
    return str(e.value)


def test_dit_messages():
    m = tpxl_b200.DiT(**TINY_DIT)
    sd = _meta(m._shapes)
    sd["x_embedder.weight"] = torch.empty(3, 3, device="meta")
    assert _raises(m, sd) == ("Error(s) in loading state_dict for DiT:\n\tsize mismatch for x_embedder.weight: copying a param with "
                              "shape (3, 3), expected (128, 8)")
    assert _raises(m, sd, strict=False).endswith("expected (128, 8)")              # a size mismatch raises without strict too
    sd = _meta(m._shapes)
    for k in list(sd)[:7]:
        del sd[k]
    sd["extra.weight"] = torch.empty(1, device="meta")
    assert _raises(m, sd) == ("Error(s) in loading state_dict for DiT:\n\tMissing key(s): ['null_cond_embedding', 'x_embedder.weight', "
                              "'x_embedder.bias', 't_embedder.mlp.0.weight', 't_embedder.mlp.0.bias']...; unexpected key(s): ['extra.weight']")
    missing, unexpected = _lib.check_state_dict("DiT", m._shapes, sd, strict=False)
    assert missing == list(m._shapes)[:7] and unexpected == ["extra.weight"]


def test_vae_messages_and_ignored_prefixes():
    v = tpxl_b200.VAE(**synth.FULL_VAE)
    sd = _meta(v._shapes)
    sd["decoder.conv_in.bias"] = torch.empty(255, device="meta")
    assert _raises(v, sd) == ("Error(s) in loading state_dict for VAE:\n\tsize mismatch for decoder.conv_in.bias: copying a param with "
                              "shape (255,), expected (256,)")
    sd = _meta(v._shapes)
    sd.update(_meta(synth.vae_encoder_shapes(**synth.FULL_VAE)))                    # encoder.* / quant_conv.* are neither
    assert _lib.check_state_dict("VAE", v._shapes, sd, True, ("encoder.", "quant_conv.")) == ([], [])
    assert _lib.check_state_dict("VAE", v._shapes, sd, False)[1] == list(synth.vae_encoder_shapes(**synth.FULL_VAE))   # without prefixes
    for k in list(v._shapes)[:6]:
        del sd[k]
    sd["decoder.bogus"] = torch.empty(1, device="meta")
    assert _raises(v, sd) == ("Error(s) in loading state_dict for VAE:\n\tMissing key(s): ['decoder.conv_in.weight', 'decoder.conv_in.bias', "
                              "'decoder.mid_block.nets.0.norm1.weight', 'decoder.mid_block.nets.0.norm1.bias', "
                              "'decoder.mid_block.nets.0.conv1.weight']...; unexpected key(s): ['decoder.bogus']")
    sd = {k: torch.zeros(s) for k, s in v._shapes.items() if k != "decoder.conv_in.bias"}
    sd["quant_conv.weight"], sd["decoder.bogus"] = torch.zeros(2, 2, 1, 1, 1), torch.zeros(1)
    res = v.load_state_dict(sd, strict=False)
    assert res.missing_keys == ["decoder.conv_in.bias"] and res.unexpected_keys == ["decoder.bogus"]
    assert list(v._extra) == ["quant_conv.weight"]


def test_dinov2_messages_after_its_own_key_steps():
    d = Dinov2Wrapper()
    bare = {k[len("model."):]: v for k, v in _meta(d._shapes).items()}           # a hub checkpoint of the bare ViT
    bare["mask_token"] = torch.empty(1, 768, device="meta")                         # dropped before the check
    bare["cls_token"] = torch.empty(1, 2, 768, device="meta")
    assert _raises(d, bare) == ("Error(s) in loading state_dict for Dinov2Wrapper:\n\tsize mismatch for model.cls_token: copying a param "
                                "with shape (1, 2, 768), expected (1, 1, 768)")
    sd = _meta(d._shapes)
    sd["model.mask_token"] = torch.empty(1, 768, device="meta")
    del sd["model.norm.bias"]
    sd["model.head.weight"] = torch.empty(1, device="meta")
    assert _raises(d, sd) == ("Error(s) in loading state_dict for Dinov2Wrapper:\n\tMissing key(s): ['model.norm.bias']; unexpected key(s): "
                              "['model.head.weight']")
    sd = {k: torch.full(s, 2.0) for k, s in d._shapes.items() if k != "model.norm.bias"}
    sd["model.mask_token"] = torch.zeros(1, 768)
    res = d.load_state_dict(sd, strict=False)
    assert res.missing_keys == ["model.norm.bias"] and res.unexpected_keys == []
    assert not d.state_dict()["model.norm.bias"].any() and bool((d.state_dict()["model.norm.weight"] == 2).all())


@pytest.fixture
def guard(monkeypatch):
    """torch.cuda.device replaced by a recorder, so that no device is needed; yields the device of each guard still open."""
    open_ = []

    @contextlib.contextmanager
    def device(dev):
        open_.append(dev)
        yield
        open_.pop()
    monkeypatch.setattr(torch.cuda, "device", device)
    return open_


class _Lib:
    """Stand-ins for tpx_*_create / tpx_*_destroy: create hands out numbered handles, destroy records what it was given."""

    def __init__(self, guard, raise_in_destroy=False):
        self.guard, self.made, self.destroyed, self.raise_in_destroy = guard, 0, [], raise_in_destroy

    def create(self, cfg, out):
        assert isinstance(cfg._obj, _lib.VaeConfig) and self.guard == ["cuda:3"]      # made under the handle's device guard
        self.made += 1
        out._obj.value = 0x1000 * self.made
        return 0

    def destroy(self, h):
        self.destroyed.append(h.value)
        if self.raise_in_destroy:
            raise RuntimeError("destroy failed")

    def handle(self):
        return _lib.Handle(self.create, self.destroy, _lib.VaeConfig(1, 6, 256, 32, 8), "cuda:3")


def test_handle_destroys_exactly_once(guard):
    lib = _Lib(guard)
    h = lib.handle()
    as_void_p = ctypes.CFUNCTYPE(ctypes.c_void_p, ctypes.c_void_p)(lambda p: p)    # what a C entry receives for the owner
    assert h.ptr.value == 0x1000 and as_void_p(h) == 0x1000 and lib.destroyed == []
    h.close()
    h.close()
    assert h.ptr is None and as_void_p(h) is None and lib.destroyed == [0x1000]
    del h
    assert lib.destroyed == [0x1000]

    class Owner:
        pass
    o = Owner()
    o.h = lib.handle()
    o.h = lib.handle()                          # replacing the owner frees the old handle
    assert lib.destroyed == [0x1000, 0x2000]
    o.h = None
    assert lib.destroyed == [0x1000, 0x2000, 0x3000]

    h = lib.handle()
    h.cycle = h                                 # only the garbage collector can free it
    del h
    gc.collect()
    assert lib.destroyed == [0x1000, 0x2000, 0x3000, 0x4000]


def test_handle_swallows_a_failing_destroy(guard):
    lib = _Lib(guard, raise_in_destroy=True)
    h = lib.handle()
    h.close()
    h.close()
    assert lib.destroyed == [0x1000] and h.ptr is None
    lib.handle()                                # dropped at once: __del__ raises nothing either
    assert lib.destroyed == [0x1000, 0x2000]


def test_scratch_grows_only():
    s = _lib.Scratch(torch.device("cpu"))
    addr, n = s.get(1000)
    buf = s.buf
    assert n == 1000 and addr % 256 == 0 and buf.data_ptr() <= addr and addr + n <= buf.data_ptr() + buf.numel()
    assert s.get(1000) == (addr, 1000) and s.buf is buf          # same size: same buffer
    assert s.get(10) == (addr, 10) and s.buf is buf              # smaller: same buffer
    addr2, n2 = s.get(100_000)
    assert n2 == 100_000 and s.buf is not buf and addr2 % 256 == 0
    assert s.buf.data_ptr() <= addr2 and addr2 + n2 <= s.buf.data_ptr() + s.buf.numel()
    assert s.get(1000) == (addr2, 1000)
