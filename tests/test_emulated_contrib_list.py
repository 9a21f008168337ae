"""CPU (kernels on the SIMT emulation, tests/emu): the compacted contribution list that the forward blend hands to the
backward (lgr_view.contrib_id_d / contrib_entry_d / contrib_count_d).  Per tile it must hold, in list order, entries of the
tile's sorted list with their ids and a non-empty set of sub-tiles -- among them every pixel's last contributor (the
forward's n_contrib), with the bit of that pixel's sub-tile, since the backward stops the pixel there."""
import numpy as np
import pytest
import torch

from oracle import torch_dense as O


@pytest.mark.parametrize('size', [(48, 32, 3000, 2.0), (64, 48, 1500, 5.0)])
def test_contribution_list_holds_every_last_contributor_in_list_order(emulated_backend, size):
    from log_b200 import GaussianRasterizationSettings, rasterize_forward
    from log_b200._capi import LGR_FILTER_MAX
    W, H, n, r = size
    cam = O.make_camera(W, H, bg=(0.1, 0.2, 0.3), dtype=torch.float32)
    sc = O.make_scene(n, W, H, r, seed=41, dtype=torch.float32)
    s = GaussianRasterizationSettings(image_height=H, image_width=W, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=cam.bg,
                                      scale_modifier=1.0, viewmatrix=cam.viewmatrix, projmatrix=cam.projmatrix, sh_degree=0,
                                      campos=cam.campos, prefiltered=False, debug=False)
    *_, st = rasterize_forward(s, sc['means3D'], sc['opacities'].reshape(-1).contiguous(), sc['scales'], sc['rotations'],
                               sc['colors'], None, LGR_FILTER_MAX, True)
    D = st.num_instances
    buf = next(t for t in st.keep if t is not None and t.data_ptr() == st.view.contrib_id_d).numpy()
    ids, entry, count = buf[:D], buf[D:2 * D].view(np.uint32), buf[2 * D:]
    start, sorted_ids, nc = st.tile_start.numpy(), st.sorted_ids.numpy(), st.n_contrib.numpy()
    assert (np.diff(start) > 256).any()          # lists that span several staged batches
    gx = (W + 15) // 16
    listed = 0
    for t in range(len(start) - 1):
        beg, ln, k = int(start[t]), int(start[t + 1] - start[t]), int(count[t])
        assert 0 <= k <= ln
        idx = (entry[beg:beg + k] >> 8).astype(np.int64)
        bits = entry[beg:beg + k] & 0xff
        assert (bits != 0).all() and (np.diff(idx) > 0).all() and (idx < ln).all()
        assert (ids[beg:beg + k] == sorted_ids[beg + idx]).all()
        ty, tx = divmod(t, gx)
        for y in range(ty * 16, min(ty * 16 + 16, H)):
            for x in range(tx * 16, min(tx * 16 + 16, W)):
                last = int(nc[y, x])
                if last == 0:
                    continue
                j = int(np.searchsorted(idx, last - 1))
                assert j < k and idx[j] == last - 1, (t, y, x)
                w = int(x % 16 >= 8) + 2 * (y % 16 // 4)          # the sub-tile (warp) of the pixel
                assert (bits[j] >> w) & 1, (t, y, x)
        listed += k
    assert 0 < listed < D
