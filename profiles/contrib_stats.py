"""How much of a tile's list would a backward that stages the whole list (up to the last contributor) stage for nothing?
One forward of a bench workload on the GPU, then, per tile, from the forward's own records (the per-tile count of the
compacted contribution list, lgr_view.contrib_count_d; n_contrib; tile_start):

  * the staged range of a full-list backward: whole 256-entry batches up to the one holding the tile's largest n_contrib;
  * the share of entries in that range that no sub-tile composited (every composited entry lies in that range, and the
    compacted list holds exactly those);
  * batches per tile when the full list is staged, and when only the compacted list is;
  * what a backward that gives every 8x4 sub-tile its own warp would walk: the (warp, splat) hits, i.e.
    the popcounts of the entries' sub-tile bytes summed, one vector RED triple per hit against one per compacted entry for a
    per-tile reduction; per tile, the slowest warp's hits over the mean of its eight warps; the compacted entries each warp
    reads (all of its tile's).

  python profiles/contrib_stats.py [--workload 10m]      (prints one JSON line)"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BATCH = 256


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='10m')
    args = ap.parse_args()
    from bench import WORKLOADS, make_inputs
    from log_b200 import GaussianRasterizationSettings, rasterize_forward
    from log_b200._capi import LGR_FILTER_MAX
    n, W, H, _, deg = WORKLOADS[args.workload]
    dev = torch.device('cuda')
    cam, sc, _ = make_inputs(args.workload)
    d = {k: v.to(dev) for k, v in sc.items()}
    settings = GaussianRasterizationSettings(
        image_height=H, image_width=W, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=cam.bg.to(dev), scale_modifier=1.0,
        viewmatrix=cam.viewmatrix.to(dev), projmatrix=cam.projmatrix.to(dev), sh_degree=deg, campos=cam.campos.to(dev),
        prefiltered=False, debug=False)
    *_, st = rasterize_forward(settings, d['means3D'], d['opacities'].reshape(-1), d['scales'], d['rotations'],
                               d['colors'] if deg == 0 else None, d['shs'] if deg > 0 else None, LGR_FILTER_MAX, True)
    torch.cuda.synchronize()
    count = st.contrib_lists()[2].cpu().numpy().astype(np.int64)
    start = st.tile_start.cpu().numpy().astype(np.int64)
    nc = st.n_contrib.cpu().numpy()
    gx, gy = (W + 15) // 16, (H + 15) // 16
    pad = np.zeros((gy * 16, gx * 16), np.int64)
    pad[:H, :W] = nc
    maxlast = pad.reshape(gy, 16, gx, 16).max(axis=(1, 3)).reshape(-1)      # per tile, in tile order
    lens = start[1:] - start[:-1]
    used = lens > 0
    # batches the backward stages: the first one always, then up to the one holding the largest n_contrib
    b_before = np.where(used, np.maximum(1, (maxlast + BATCH - 1) // BATCH), 0)
    staged = np.minimum(lens, b_before * BATCH)
    nz_staged = count[:len(lens)]
    assert (nz_staged <= staged).all()
    b_after = (nz_staged + BATCH - 1) // BATCH
    # per (tile, sub-tile) hits of the compacted lists: bit w of an entry's low byte = sub-tile w composited it
    entry = st.contrib_lists()[1].cpu().numpy().view(np.uint32)
    ntiles = len(lens)
    cnt = nz_staged
    pos = np.repeat(start[:ntiles], cnt) + (np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt))
    byte = (entry[pos] & 0xff).astype(np.uint8)
    bits = np.unpackbits(byte[:, None], axis=1, bitorder='little')                  # (entries, 8): bit w
    tile_of = np.repeat(np.arange(ntiles), cnt)
    hits_tw = np.zeros((ntiles, 8), np.int64)
    np.add.at(hits_tw, tile_of, bits.astype(np.int64))
    busy = hits_tw.sum(axis=1) > 0
    imb = hits_tw[busy].max(axis=1) / hits_tw[busy].mean(axis=1)
    hits = int(hits_tw.sum())
    out = {
        'workload': args.workload, 'gpu': torch.cuda.get_device_name(), 'instances': int(lens.sum()),
        'tiles': int(len(lens)), 'tiles_with_entries': int(used.sum()),
        'staged_entries': int(staged.sum()), 'nonzero_staged_entries': int(nz_staged.sum()),
        'zero_share_of_staged': float(1.0 - nz_staged.sum() / max(staged.sum(), 1)),
        'staged_share_of_list': float(staged.sum() / max(lens.sum(), 1)),
        'batches_per_tile_before': {'mean': float(b_before[used].mean()), 'max': int(b_before.max()), 'total': int(b_before.sum())},
        'batches_per_tile_after': {'mean': float(b_after[used].mean()), 'max': int(b_after.max()), 'total': int(b_after.sum())},
        'warp_hits': hits, 'warp_hits_per_entry': float(hits / max(int(cnt.sum()), 1)),
        'vector_reds': {'per_warp_hit': 3 * hits, 'per_entry': 3 * int(cnt.sum())},
        'slowest_warp_over_mean': {'mean': float(imb.mean()), 'p50': float(np.median(imb)), 'p90': float(np.percentile(imb, 90)),
                                   'hit_weighted': float((hits_tw[busy].max(axis=1) * 8).sum() / max(hits, 1))},
        'entries_per_warp_tile': {'mean': float(cnt[busy].mean()), 'max': int(cnt.max()),
                                  'hits_per_warp_tile_mean': float(hits_tw[busy].mean())},
    }
    print(json.dumps(out))


if __name__ == '__main__':
    main()
