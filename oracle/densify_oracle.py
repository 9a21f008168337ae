"""TEST INFRASTRUCTURE ONLY -- torch restatement of LoG's Splitter.split_and_remove / split_and_remove_other
(LoG/model/splitter.py:95-220, geometry.py:4-25), the checker for log_b200/csrc/lgr_densify.cu.  Only tests/ and
profiles/ may import this.

Runs on any device.  `copy_device=None` rebuilds the tables where they are; `copy_device='cpu'` makes LoG's round trip
through host memory (tables and optimiser state to the CPU, rebuilt there, back), which is what the benchmark times.
split_by_uniform's 3x3 matmul is written as the one product it reduces to (the other two offsets are zero), so the
rounding does not depend on a BLAS.  Pinned bit for bit against LoG's own Splitter run on CPU tensors
(tests/golden/reference_densify.npz, made by tests/golden/make_densify_golden.py)."""
import torch


def build_rotation(r):
    """geometry.py:4-25, each operation rounded once."""
    norm = torch.sqrt(r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1] + r[:, 2] * r[:, 2] + r[:, 3] * r[:, 3])
    q = r / norm[:, None]
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    return torch.stack([torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                        torch.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
                        torch.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def split_by_uniform(xyz, scaling_raw, rotation_raw, N):
    """splitter.py:95-130 for the split parents' raw rows -> (children xyz (N S, 3), children raw scaling (N S, 3),
    the four printed means as 0-d tensors: parent scale, parent max scale, child scale, child max scale)."""
    S = xyz.shape[0]
    s = torch.exp(scaling_raw)
    stats = [s.mean(), s.max(dim=-1).values.mean()]
    R = build_rotation(rotation_raw)
    rows = torch.arange(S, device=xyz.device)
    c = xyz[:, None]
    for _ in range(N.bit_length() - 1):
        k = s.max(dim=-1).indices                               # first index on ties
        d = R[rows, :, k] * (0.5 * s[rows, k])[:, None]         # R @ (+-0.5 s_k e_k): one product per row
        c = torch.stack([c + (-d)[:, None], c + d[:, None]], dim=2).reshape(S, -1, 3)
        s = s.clone()
        s[rows, k] *= 0.5
    s = s[:, None].expand(S, N, 3).reshape(-1, 3)
    stats += [s.mean(), s.max(dim=-1).values.mean()]
    return c.reshape(-1, 3), torch.log(s), stats


def split_and_remove(splitter, model, optimizer, flag_split, flag_remove, remove_split=True, copy_device=None):
    """splitter.py:138-205 with split_method 'uniform'; returns num_keep (0-d on the flags' device)."""
    N = splitter.N
    print(f'[{splitter.__class__.__name__}] split method {splitter.split_method}, remove {flag_split.shape[0]} '
          f'+{flag_split.sum()}x{N} -{flag_remove.sum()}')
    split_info = {}
    if flag_split.sum() > 0:
        index = torch.where(flag_split)[0]
        cxyz, cscaling, stats = split_by_uniform(model.xyz[index].detach(), model.scaling[index].detach(),
                                                 model.rotation[index].detach(), N)
        split_info = {'xyz': cxyz, 'scaling': cscaling}
        name = model.__class__.__name__
        print(f'[{name}] split : {flag_split.sum()} -> {cxyz.shape[0]}')
        print(f'[{name}] radius: {stats[0].item():.4f} -> {stats[2].item():.4f}, {stats[1].item():.4f} -> {stats[3].item():.4f}')
    if remove_split:
        flag_remove = flag_remove | flag_split
    num_keep = (~flag_remove).sum()
    dev = copy_device or flag_split.device
    keep, split = (~flag_remove).to(dev), flag_split.to(dev)
    for key in model.keys:
        old = getattr(model, key, None)
        if old is None or old.shape[0] == 0:
            continue
        origin = old.device
        old = old.detach().to(dev)
        parts = [old[keep]]
        if split.any():
            parts.append(split_info[key].to(dev) if key in split_info else
                         old[split][:, None].repeat(1, N, *[1] * (old.dim() - 1)).reshape(-1, *old.shape[1:]))
        with torch.no_grad():
            getattr(model, key).set_(torch.cat(parts, dim=0).to(origin))
    if optimizer is None:
        return num_keep
    for state_key in optimizer.state_keys:
        for key, val in getattr(optimizer, state_key).items():
            origin = val.device
            old = val.to(dev)
            new = getattr(model, key)
            zeros = torch.zeros((new.shape[0] - old[keep].shape[0], *old.shape[1:]), dtype=old.dtype, device=dev)
            val.set_(torch.cat([old[keep], zeros], dim=0).to(origin))
    return num_keep


def split_and_remove_other(splitter, model, keys, flag_split, flag_remove, remove_split=True):
    """splitter.py:207-220."""
    if remove_split:
        flag_remove = flag_remove | flag_split
    num_keep = (~flag_remove).sum()
    for key in keys:
        old = getattr(model, key, None)
        if old is None or old.shape[0] == 0:
            continue
        new = torch.zeros((num_keep + flag_split.sum() * splitter.N,), device=old.device, dtype=old.dtype)
        new[:num_keep] = old[~flag_remove]
        if key == 'radius3d_min':
            new[num_keep:] = old[flag_split][:, None].repeat(1, splitter.N).reshape(-1)
        old.set_(new)
