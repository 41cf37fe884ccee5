"""Host (numpy) restatement of empty-space skipping (csrc/occupancy.cu): the cell reduction of the node alphas, the box
dilation, the bit packing and the per-group tile ranges of a ray launch.  The CPU tests pin it on hand-made inputs; the
GPU tests compare the kernels with it."""
import numpy as np


def cells_from_alpha(alpha):
    """alpha [D,Hp,Wp] at the nodes -> bool [D,Hp,Wp]: cell (d,y,x) (d < D-1, y < Hp-1, x < Wp-1) set when alpha > 0 at
    any of its eight corner nodes; the last slab of each axis is False."""
    pos = np.asarray(alpha) > 0
    D, H, W = pos.shape
    out = np.zeros_like(pos)
    c = np.zeros((D - 1, H - 1, W - 1), dtype=bool)
    for dz in (0, 1):
        for dy in (0, 1):
            for dx in (0, 1):
                c |= pos[dz:D - 1 + dz, dy:H - 1 + dy, dx:W - 1 + dx]
    out[:D - 1, :H - 1, :W - 1] = c
    return out


def dilate(cells, r):
    """box dilation by r cells over the valid cells (the last slab of each axis stays False)"""
    cells = np.asarray(cells, dtype=bool)
    D, H, W = cells.shape
    v = cells[:D - 1, :H - 1, :W - 1]
    for axis in range(3):
        acc = np.zeros_like(v)
        n = v.shape[axis]
        for k in range(-r, r + 1):
            src = [slice(None)] * 3
            dst = [slice(None)] * 3
            if k >= 0:
                src[axis], dst[axis] = slice(k, n), slice(0, n - k)
            else:
                src[axis], dst[axis] = slice(0, n + k), slice(-k, n)
            acc[tuple(dst)] |= v[tuple(src)]
        v = acc
    out = np.zeros_like(cells)
    out[:D - 1, :H - 1, :W - 1] = v
    return out


def pack(cells):
    """bool [D,Hp,Wp] -> int32 words, bit c = linear index c of word c // 32, LSB first"""
    flat = np.asarray(cells, dtype=bool).reshape(-1)
    n = (flat.size + 31) // 32 * 32
    padded = np.zeros(n, dtype=np.uint64)
    padded[:flat.size] = flat
    words = (padded.reshape(-1, 32) << np.arange(32, dtype=np.uint64)).sum(1)
    return words.astype(np.uint32).view(np.int32)


def unpack(words, shape):
    w = np.asarray(words).view(np.uint32).astype(np.uint64)
    bits = (w[:, None] >> np.arange(32, dtype=np.uint64)) & 1
    return bits.reshape(-1)[:int(np.prod(shape))].astype(bool).reshape(shape)


def sample_occupied(ndc, cells):
    """ndc [..., 3] (x, y, z) fp32 -> bool [...]: outside [0,1]^3 (or NaN) counts as occupied, otherwise the bit of the
    cell whose lower corner is floor of the trilinear index, clamped to the last cell (the kernel's arithmetic)."""
    ndc = np.asarray(ndc, dtype=np.float32)
    D, H, W = cells.shape
    nx, ny, nz = ndc[..., 0], ndc[..., 1], ndc[..., 2]
    with np.errstate(invalid="ignore"):
        inside = (nx >= 0) & (nx <= 1) & (ny >= 0) & (ny <= 1) & (nz >= 0) & (nz <= 1)
    one, half = np.float32(1), np.float32(0.5)

    def idx(n, size):
        i = ((n * np.float32(2) - one + one) * half) * np.float32(size - 1)
        return np.clip(np.floor(np.where(inside, i, 0)).astype(np.int64), 0, size - 2)
    x, y, z = idx(nx, W), idx(ny, H), idx(nz, D)
    return ~inside | cells[z, y, x]


def rays_per_tile(n, sms):
    """the render launcher's rule: 32 unless the batch gives fewer than two groups per SM"""
    rt = 32
    while rt > 4 and (n + rt - 1) // rt < 2 * sms:
        rt //= 2
    return rt


def group_ranges(occupied, rt):
    """occupied [N,S] bool -> int [G,2] = (k_first, k_last) per group of rt rays, tile = sample // (64 // rt);
    (NT, -1) when no sample of the group is occupied."""
    occupied = np.asarray(occupied, dtype=bool)
    N, S = occupied.shape
    sp = 64 // rt
    nt = (S + sp - 1) // sp
    G = (N + rt - 1) // rt
    out = np.empty((G, 2), dtype=np.int64)
    tiles = np.arange(S) // sp
    for g in range(G):
        t = tiles[occupied[g * rt:(g + 1) * rt].any(0)]
        out[g] = (t.min(), t.max()) if t.size else (nt, -1)
    return out
