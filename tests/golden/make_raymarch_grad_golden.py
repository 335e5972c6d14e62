#!/usr/bin/env python
"""Golden vectors for the ray-march GRADIENTS, produced by running the reference's own pure-PyTorch ray-marcher under autograd.

Run in the build container only (needs /root/reference):

    python tests/golden/make_raymarch_grad_golden.py

The reference's gradcheck (mvpraymarch.py:301-559) checks its CUDA backward against autograd through the plain PyTorch block under
"# python raymarching implementation".  As in make_raymarch_golden.py, that block is read from the reference file AT RUN TIME (nothing
of it is stored here) and executed on the CPU, here with template / primpos / primrot / primscale as leaf tensors that require grad;
``rayrgba.backward(G)`` with a seeded upstream G (not all ones, so the four channels are told apart) gives the four gradients.  Two
scenes: the sparse scene of raymarch_ref.npz, and a dense one where more than 10 % of the rays saturate and more than 20 % are covered
but unsaturated (the saturation term of the backward is the part that is easy to get wrong).

The file also holds the pixel coordinates of the reference's subsample_pixel_coords (training) and resize_pixel_coords (eval), read
from dva/ray_marcher.py at run time, for f in {2, 3, 4}, B = 3, after torch.manual_seed(1234).  Everything goes to
tests/golden/raymarch_grad.npz; tests/test_raymarch_grad_host.py holds the oracle and the host offset draw to it.
"""
import ast
import importlib.util
import os

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "raymarch_grad.npz")
REF_RAY_MARCHER = "/root/reference/dva/ray_marcher.py"
PIX_SEED, PIX_B, PIX_H, PIX_W = 1234, 3, 14, 11


def _forward_golden():
    spec = importlib.util.spec_from_file_location("make_raymarch_golden", os.path.join(HERE, "make_raymarch_golden.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def dense_scene(base):
    sc = base.scene(seed=11, H=16, W=16, K=10, M=6)
    sc["template"][:, :, 3] *= 1.5
    sc["primscale"] = sc["primscale"] * 1.2
    sc["fadescale"], sc["fadeexp"] = 6.5, 7.5          # the reference gradcheck's own fade (mvpraymarch.py:555-557)
    return sc


def run(base, sc, seed):
    leaves = {k: sc[k].clone().requires_grad_(True) for k in ("template", "primpos", "primrot", "primscale")}
    ns = dict(sc)
    ns.update(leaves)
    ns.update(torch=torch, F=F, dowarp=False, accum=0, warp=None)
    exec(compile(base.reference_block(), base.REF_FILE + ":<python raymarching block>", "exec"), ns)
    out = ns["rayrgba"]
    G = torch.randn(out.shape, generator=torch.Generator().manual_seed(seed))
    out.backward(G)
    alpha = out.detach()[..., 3]
    sat = float((alpha >= 1.0 - 1e-6).float().mean())
    cov_unsat = float(((alpha > 0) & (alpha < 1.0 - 1e-6)).float().mean())
    print(f"steps {ns['step']}, saturated {sat:.2f}, covered but unsaturated {cov_unsat:.2f}")
    return out.detach(), G, {k: v.grad for k, v in leaves.items()}, sat, cov_unsat


def pixel_coords():
    """The two helpers' sources from dva/ray_marcher.py, executed as they stand (the module itself imports the sm_70 extensions)."""
    tree = ast.parse(open(REF_RAY_MARCHER).read())
    ns = {"th": torch}
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name in ("subsample_pixel_coords", "resize_pixel_coords"):
            exec(compile(ast.Module([node], []), REF_RAY_MARCHER, "exec"), ns)
    base = torch.stack(torch.meshgrid(torch.arange(PIX_H, dtype=torch.float32), torch.arange(PIX_W, dtype=torch.float32), indexing="ij")[::-1], dim=-1)
    out = {}
    torch.manual_seed(PIX_SEED)
    for f in (2, 3, 4):
        out[f"pix_train_f{f}"] = ns["subsample_pixel_coords"](base, PIX_B, f).numpy()
        out[f"pix_eval_f{f}"] = ns["resize_pixel_coords"](base, PIX_B, f).numpy()
    return out


def main():
    base = _forward_golden()
    arrays = {}
    for name, sc, seed in (("sparse", base.scene(), 21), ("dense", dense_scene(base), 22)):
        out, G, grads, sat, cov_unsat = run(base, sc, seed)
        if name == "dense":
            assert sat > 0.10 and cov_unsat > 0.20, (sat, cov_unsat)
        arrays.update({
            f"{name}_raypos": sc["raypos"].numpy(), f"{name}_raydir": sc["raydir"].numpy(), f"{name}_tminmax": sc["tminmax"].numpy(),
            f"{name}_stepsize": np.float32(sc["stepsize"]), f"{name}_fadescale": np.float32(sc["fadescale"]), f"{name}_fadeexp": np.float32(sc["fadeexp"]),
            f"{name}_template_chlast": sc["template"].permute(0, 1, 3, 4, 5, 2).contiguous().numpy(),
            f"{name}_primpos": sc["primpos"].numpy(), f"{name}_primrot": sc["primrot"].numpy(), f"{name}_primscale": sc["primscale"].numpy(),
            f"{name}_rayrgba": out.numpy(), f"{name}_grad_rayrgba": G.numpy(),
            f"{name}_grad_template_chlast": grads["template"].permute(0, 1, 3, 4, 5, 2).contiguous().numpy(),
            f"{name}_grad_primpos": grads["primpos"].numpy(), f"{name}_grad_primrot": grads["primrot"].numpy(),
            f"{name}_grad_primscale": grads["primscale"].numpy()})
    arrays.update(pixel_coords())
    arrays.update(pix_seed=np.int64(PIX_SEED), pix_hw=np.array([PIX_B, PIX_H, PIX_W]))
    np.savez_compressed(OUT, **arrays)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
