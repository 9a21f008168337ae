"""The C ABI's answer to every colour-source combination of lgr_forward_project and lgr_backward.

Which colour source a call has -- precomputed (N,3) or (N,6) colours, stock SH, LoG's raw DC + rest coefficients -- with
or without cov3D_precomp, the depth pass, band mode or a gather index, is decided from the view and from which pointers
are null.  This test pins the return code of both entry points over the whole matrix below (n = 16 on a 32x32 view)
against tests/golden/colour_source_abi.json, so that the way the decision is made can change while every answer stays:
'0' accepted (the kernels ran), 'B' LGR_E_BADARG, 'U' LGR_E_UNSUPPORTED.  The table is `table()` of the library as it was
before the colour source became one enum (lgr::Colour), written out as JSON with the axes.  Every buffer has its real
size; the backward takes the forward's radii, so its kernel runs the full chain rule exactly for the cases the forward
accepted.
"""
import ctypes
import itertools
import json
import os

import torch

from test_render_depth import BG, cov6, make, settings
from test_six_channels import backend  # noqa: F401  (the fixture: H100 and CPU emulation)

N, W, H = 16, 32, 32
AXES = {'colours': (3, 6, None), 'shs': (0, 1), 'raw_params': (0, 1), 'cov3D_precomp': (0, 1),
        'channels_log_depth': ((3, 0), (3, 1), (6, 0), (6, 1)), 'band': (0, 1), 'gather': (0, 1), 'sh_degree': (0, 3, 4),
        'sh_coeffs': ('short', 'exact')}
CODES = {0: '0', -1: 'B', -3: 'U'}
ROW = 4 * 2 * 2 * 3 * 2      # cases per line of the table: one line per (colours, shs, raw_params, cov3D_precomp)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'colour_source_abi.json')


def run_case(lib, dev, cam, sc, colours, shs, raw, cov3d, channels, band, gather, deg, coeffs):
    """(forward return code, backward return code) of one case."""
    from log_b200._capi import LGR_FILTER_MAX, LGR_GRAD_FLOATS, LGR_META_INTS, LGR_ROW_FLOATS, LGR_SPLAT_FLOATS, \
        LGR_TILE_SCRATCH_INTS
    from log_b200.rasterizer import _make_view
    nc, log_depth = channels
    f32, i32 = dict(dtype=torch.float32, device=dev), dict(dtype=torch.int32, device=dev)
    z = lambda *s, **kw: torch.zeros(*s, **(kw or f32))
    P = lambda x: None if x is None else ctypes.c_void_p(x.data_ptr())
    t = {k: v.to(**f32).contiguous() for k, v in sc.items()}
    # exact = what the layout needs: (deg+1)^2 stock coefficients, or the (deg+1)^2 - 1 rest coefficients of LoG's layout
    K = (deg + 1) ** 2 - (1 if raw and colours else 0) - (coeffs == 'short')
    # lgr_view cannot tell (N,3) colours from (N,6): both live in (N,6) storage, so a call that reads six stays in bounds
    col = None
    if colours:
        col = z(N * 6)[:N * colours].view(N, colours)
        col[:, :3] = t['colors']
    sh = z(N * max(K, 1) * 3) if shs else None
    cov = cov6(sc).to(**f32) if cov3d else None
    ntiles = ((W + 15) // 16) * ((H + 15) // 16)
    band = dict(num_owners=2, band_ids=z(256, **i32), band_count=z(2, **i32), band_blk=z(3, **i32),
                band_rows=z(N, **i32)) if band else {}
    index = torch.randperm(N, generator=torch.Generator().manual_seed(1)).to(dev) if gather else None
    ext, dcov = z(N, 4), z(N, 6)
    keep = [cov, index, ext, dcov, *band.values()]      # the view holds raw pointers
    v = _make_view(settings(cam, dev, deg, bg=BG * (nc // 3)), LGR_FILTER_MAX, False, K, (0, 1) if band else None, keep,
                   raw_params=raw, gather_index=index, cov3D_precomp=cov, **band)
    v.num_channels, v.log_depth = nc, log_depth
    v.splat_ext_d = ext.data_ptr() if nc == 6 else None
    v.dcov3D_d = dcov.data_ptr() if cov3d else None
    splat, radii, clamped = z(N * LGR_SPLAT_FLOATS), z(N, **i32), z(N, dtype=torch.uint8, device=dev)
    tile_start, cursor, meta = z(ntiles + 1, **i32), z(LGR_TILE_SCRATCH_INTS * ntiles, **i32), z(LGR_META_INTS, **i32)
    image, dimage, dsplat = z(nc, H, W), z(nc, H, W) + 0.1, z(N * LGR_GRAD_FLOATS) + 0.01
    grads = [z(N, 3), z(N, 3), z(N), z(N, 3), z(N, 4), z(N * 6), z(N * max(K, 1) * 3), z(N * LGR_ROW_FLOATS) if band else None]
    inputs = [t['means3D'], t['opacities'], t['scales'], t['rotations'], col, sh]
    fwd = lib.lgr_forward_project(ctypes.byref(v), N, *map(P, inputs + [splat, radii, clamped, tile_start, cursor, meta]), None)
    bwd = lib.lgr_backward(ctypes.byref(v), N, 0, *map(P, inputs + [splat, radii, clamped, tile_start, None, image, dimage, dsplat]
                                                       + grads), None, 0, N, None)
    return fwd, bwd


def table(lib, dev):
    """{'forward': [...], 'backward': [...]}: one character per case, in the order of itertools.product over AXES."""
    cam, sc = make(W, H, N, 3.0, seed=2)
    out = {'forward': '', 'backward': ''}
    for case in itertools.product(*AXES.values()):
        for name, rc in zip(out, run_case(lib, dev, cam, sc, *case)):
            assert rc in CODES, f'{name} {dict(zip(AXES, case))}: return code {rc}'
            out[name] += CODES[rc]
    if dev.type == 'cuda':
        torch.cuda.synchronize(dev)
        torch.cuda.empty_cache()      # ~40k small buffers: leave the allocator to later tests as we found it
    return {k: [s[i:i + ROW] for i in range(0, len(s), ROW)] for k, s in out.items()}


def test_colour_source_return_codes(backend):
    from log_b200 import _capi
    with open(GOLDEN) as fh:
        want = json.load(fh)
    assert want['axes'] == [[k, [list(x) if isinstance(x, tuple) else x for x in v]] for k, v in AXES.items()]
    got = table(_capi.load(), backend)
    cases = list(itertools.product(*AXES.values()))
    bad = [(name, dict(zip(AXES, cases[i])), w, g) for name in ('forward', 'backward')
           for i, (w, g) in enumerate(zip(''.join(want[name]), ''.join(got[name]))) if w != g]
    assert not bad, f'{len(bad)} cases changed, e.g. (entry point, case, expected, got): {bad[:8]}'

