"""-m gpu: the box-projection unwrap and noise filter (csrc/uv_unwrap.cu through tpxl_b200.unwrap) against the oracle, fed with the
kernels' own previous stage, and against the reference's outputs (tests/golden/unwrap.npz); determinism; edge inputs;
PrimSDF.extract_texmesh against the explicit chain."""
import os

import numpy as np
import pytest
import torch

from oracle import unwrap as ou
from tpxl_b200 import unwrap

from test_gpu_mesh import _shell_module
from test_unwrap_host import MESHES, ROT_TOL

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "unwrap.npz")


def _run(v, f, pad=0.02):
    dv, df = torch.from_numpy(np.ascontiguousarray(v, np.float32)).cuda(), torch.from_numpy(np.ascontiguousarray(f, np.int64)).cuda()
    n = unwrap.compute_vertex_normal(dv, df)
    taps = {}
    uv, vidx = unwrap.box_projection_uv_unwrap(dv, n, df, pad, taps=taps)
    return n.cpu().numpy(), {k: t.cpu().numpy() for k, t in taps.items()}, uv.cpu().numpy(), vidx.cpu().numpy()


def _check_stages(v, f, n, t, uv, vidx, pad=0.02):
    np.testing.assert_allclose(n, ou.vertex_normals(v, f), rtol=0, atol=1e-6)
    slc, fuv, pm = ou.project(v, n, f)
    assert ((t["slice"] == slc) | (pm < 1e-6)).all()
    same = t["slice"] == slc
    np.testing.assert_allclose(t["face_uv"][same], fuv[same], rtol=0, atol=1e-6)
    ang, ruv = ou.rotate(v, n, f, t["face_uv"], t["slice"])
    np.testing.assert_allclose(t["rot_uv"], ruv, rtol=0, atol=2e-6)
    asg, mk = ou.assign(v, f, t["rot_uv"], t["slice"])
    assert ((t["assign"] == asg) | ou.ambiguous(mk)).all()
    np.testing.assert_allclose(t["placed"], ou.place(t["rot_uv"], t["assign"], pad), rtol=0, atol=1e-6)
    u2, i2 = ou.unique(t["placed"])
    assert np.array_equal(uv, u2) and np.array_equal(vidx, i2)
    assert np.array_equal(uv[vidx], t["placed"])
    assert uv.min() >= 0 and uv.max() <= 1
    assert ou.residual_overlaps(t["rot_uv"], t["assign"]) == 0


@pytest.mark.parametrize("name", MESHES)
def test_stages_match_oracle_and_reference(name):
    g = np.load(GOLDEN)
    v, f = g[f"{name}_v"], g[f"{name}_f"].astype(np.int64)
    n, t, uv, vidx = _run(v, f)
    _check_stages(v, f, n, t, uv, vidx)
    # end to end against the reference: equal decisions, per-corner uv within the rotation stage's bound
    assert np.array_equal(t["slice"], g[f"{name}_slice"]) and np.array_equal(t["assign"], g[f"{name}_assign"])
    np.testing.assert_allclose(uv[vidx], g[f"{name}_placed"], rtol=0, atol=ROT_TOL)


def test_shell_and_determinism():
    """extract_mesh(256, 8, 0.05, 100000) of the shell: atlas invariants on the kernels' own outputs (the oracle's kd-tree is not run:
    the decimated mesh's long UV slivers give it near-quadratic candidate lists), and identical bytes on repeats and a side stream."""
    m = _shell_module()
    v, f = m.extract_mesh(256, min_faces=8, min_diameter=0.05, target_faces=100000)
    print("mesh", v.shape[0], f.shape[0], flush=True)
    n = unwrap.compute_vertex_normal(v, f)
    taps = {}
    uv, vidx = unwrap.box_projection_uv_unwrap(v, n, f, 0.02, taps=taps)
    torch.cuda.synchronize()
    print("unwrap", uv.shape[0], flush=True)
    placed, asg = taps["placed"].cpu().numpy(), taps["assign"].cpu().numpy()
    assert np.array_equal(uv.cpu().numpy()[vidx.cpu().numpy()], placed)
    assert float(uv.min()) >= 0 and float(uv.max()) <= 1 and (np.diff(uv.cpu().numpy()[:, 0]) >= 0).all()
    cell = ou.slot_cells(asg)
    assert (placed[..., 0] >= cell[:, None, 0] - 1e-6).all() and (placed[..., 0] <= cell[:, None, 2] + 1e-6).all()
    assert (placed[..., 1] >= cell[:, None, 1] - 1e-6).all() and (placed[..., 1] <= cell[:, None, 3] + 1e-6).all()
    assert ((asg == taps["slice"].cpu().numpy()) | (asg >= 6)).all()
    again = unwrap.box_projection_uv_unwrap(v, n, f.int(), 0.02)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        n2 = unwrap.compute_vertex_normal(v, f)
        other = unwrap.box_projection_uv_unwrap(v, n2, f, 0.02)
    torch.cuda.current_stream().wait_stream(side)
    assert torch.equal(n2, n)
    for a, b in (again, other):
        assert torch.equal(a, uv) and torch.equal(b, vidx)


def _edge_cases():
    rs = np.random.RandomState(3)
    one = (np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0.1]], np.float32), np.array([[0, 1, 2]]))
    xs, ys = np.meshgrid(np.linspace(0, 1, 30), np.linspace(0, 1, 30), indexing="ij")
    grid_v = np.stack([xs.ravel(), ys.ravel(), 0.001 * rs.standard_normal(900)], 1).astype(np.float32)
    q = (np.arange(29)[:, None] * 30 + np.arange(29)[None]).ravel()
    flat_f = np.concatenate([np.stack([q, q + 30, q + 1], 1), np.stack([q + 1, q + 30, q + 31], 1)])
    zero_f = np.concatenate([flat_f, [[0, 0, 1], [5, 5, 5]]])                  # zero-area faces with repeated indices
    huge_v = np.concatenate([grid_v, [[-0.1, -0.1, 0.01], [2.0, -0.1, 0.01], [-0.1, 2.0, 0.01]]]).astype(np.float32)
    huge_f = np.concatenate([flat_f, [[900, 901, 902]]])                      # one triangle over all the small ones
    dup_f = np.concatenate([flat_f, flat_f[:50], flat_f[:50]])              # coincident centroids
    return {"one": one, "one_slice": (grid_v, flat_f), "zero_area": (grid_v, zero_f), "huge": (huge_v, huge_f), "coincident": (grid_v, dup_f)}


@pytest.mark.parametrize("case", sorted(_edge_cases()))
def test_edge_inputs(case):
    v, f = _edge_cases()[case]
    n, t, uv, vidx = _run(v, f)
    _check_stages(v, f.astype(np.int64), n, t, uv, vidx)
    if case == "one_slice":
        assert (t["slice"] % 6 == t["slice"][0] % 6).all()


def test_bad_input_raises():
    v = torch.rand(4, 3, device="cuda")
    n = unwrap.compute_vertex_normal(v, torch.tensor([[0, 1, 2]], device="cuda"))
    for bad in ([[0, 1, 4]], [[-1, 1, 2]]):
        with pytest.raises(ValueError):
            unwrap.box_projection_uv_unwrap(v, n, torch.tensor(bad, device="cuda"), 0.02)
        with pytest.raises(ValueError):
            unwrap.compute_vertex_normal(v, torch.tensor(bad, device="cuda"))
    with pytest.raises(ValueError):
        unwrap.box_projection_uv_unwrap(v, n, torch.tensor([[0, 1, 2]], device="cuda"), 0.6)
    with pytest.raises(unwrap._lib.TpxError):
        unwrap.compute_vertex_normal(v.cpu(), torch.tensor([[0, 1, 2]]))


def test_noise_filter():
    g = np.load(GOLDEN)
    for name in ("dense", "spread"):
        keep, nn = unwrap.noise_filter(torch.from_numpy(g[f"noise_{name}_srt"]).cuda(), return_nn=True)
        assert np.array_equal(keep.cpu().numpy(), g[f"noise_{name}_keep"]) and np.array_equal(nn.cpu().numpy(), g[f"noise_{name}_nn"])
    m = _shell_module()
    k, o = m.noise_filter_mask().cpu().numpy(), ou.noise_filter(m.srt_param.detach().cpu().numpy())[0]
    assert m.srt_param.shape[0] == 2048 and np.array_equal(k, o)


def test_extract_texmesh_equals_explicit_chain():
    m = _shell_module()
    before = m.srt_param.detach().clone()
    out = m.extract_texmesh(resolution=128, target_faces=20000, atlas=256)
    assert torch.equal(m.srt_param.detach(), before)
    keep = m.noise_filter_mask()
    from tpxl_b200 import PrimSDF
    sub = PrimSDF(num_prims=0)
    sub.srt_param.data, sub.feat_param.data = m.srt_param.detach()[keep].contiguous(), m.feat_param.detach()[keep].contiguous()
    sub.eval()
    v, f = sub.extract_mesh(128, min_faces=8, min_diameter=0.05, target_faces=20000)
    uv, idx = unwrap.box_projection_uv_unwrap(v, unwrap.compute_vertex_normal(v, f), f, 0.02)
    vt = uv[idx].reshape(-1, 2)
    ft = torch.arange(3 * f.shape[0], device="cuda").reshape(-1, 3)
    feats, mask = sub.bake_texture(v[f].reshape(-1, 3), ft, vt, ft, 256)
    assert torch.equal(out["v"], v) and torch.equal(out["f"], f) and torch.equal(out["vt"], vt) and torch.equal(out["ft"], ft)
    assert torch.equal(out["albedo"], feats[..., :3] / 255) and torch.equal(out["metallicRoughness"], feats[..., 3:] / 255)
    assert mask.float().mean() > 0.1 and out["albedo"].min() >= 0 and out["albedo"].max() <= 1
