#!/usr/bin/env python
"""Golden vectors for deep kernel learning (gp_ski_input_grad, gpytorch_b200.utils.grid.ScaleToBounds), produced by EXECUTING the
reference's own code, loaded as make_golden_ski.py loads it:
  * d(interp_values)/dx from autograd through Interpolation.interpolate (utils/interpolation.py:44-167) in fp64, for interior
    points, points in the one-hot first / last cells and points exactly on grid nodes;
  * ScaleToBounds (utils/grid.py:11-54) outputs in train and eval mode and the gradient of a weighted sum of the training output.
Output: tests/golden/dkl_golden.npz (committed).  Re-run:  python tests/golden/make_golden_dkl.py
"""
import os

import numpy as np
import torch

from make_golden_ski import HERE, load_reference


def main():
    grid_mod, Interpolation = load_reference()
    out = {}
    for tag, sizes, npts in (("d1", [20], 30), ("d2", [12, 15], 40), ("d3", [8, 9, 10], 30)):
        d = len(sizes)
        g = torch.Generator().manual_seed(501 + d)
        grid = grid_mod.create_grid(sizes, [(0.0, 1.0)] * d, extend=True, dtype=torch.float64)
        x = torch.rand(npts, d, generator=g, dtype=torch.float64)
        for i, gax in enumerate(grid):
            h = float(gax[1] - gax[0])
            x[0, i] = gax[0] + 0.4 * h          # first cell (one-hot)
            x[1, i] = gax[-2] + 0.3 * h         # last cell (one-hot)
            x[2, i] = gax[3]                    # on an interior node
            x[3, i] = gax[1]                    # on the node that closes the first cell
            x[4, i] = gax[-2]                   # on the node that opens the last cell
        xr = x.clone().requires_grad_(True)
        idx, val = Interpolation().interpolate(grid, xr)
        dval = torch.zeros(d, *val.shape, dtype=torch.float64)
        for q in range(val.size(1)):
            (gq,) = torch.autograd.grad(val[:, q].sum(), xr, retain_graph=True)
            dval[:, :, q] = gq.t()
        out[f"{tag}_x"] = x.numpy()
        for i, gax in enumerate(grid):
            out[f"{tag}_grid{i}"] = gax.numpy()
        out[f"{tag}_idx"] = idx.numpy()
        out[f"{tag}_val"] = val.detach().numpy()
        out[f"{tag}_dval"] = dval.numpy()
    m = grid_mod.ScaleToBounds(-1.0, 1.0).double()
    g = torch.Generator().manual_seed(9)
    xt = (3.0 * torch.randn(25, 2, generator=g, dtype=torch.float64) + 0.5).requires_grad_(True)
    wt = torch.randn(25, 2, generator=g, dtype=torch.float64)
    m.train()
    yt = m(xt)
    (gx,) = torch.autograd.grad((yt * wt).sum(), xt)
    xe = 5.0 * torch.randn(10, 2, generator=g, dtype=torch.float64)
    m.eval()
    out.update(stb_x=xt.detach().numpy(), stb_w=wt.numpy(), stb_train=yt.detach().numpy(), stb_grad=gx.numpy(),
               stb_xe=xe.numpy(), stb_eval=m(xe).detach().numpy())
    np.savez_compressed(os.path.join(HERE, "dkl_golden.npz"), **out)
    print("wrote", len(out), "arrays")


if __name__ == "__main__":
    main()
