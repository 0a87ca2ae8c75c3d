"""Plain restatements of the index-deciding rules, and generators of inputs that sit exactly on their decision boundaries.

* The lookup's cells (k_corr_lookup and k_lookup_bwd): offset d = fl(x - c), quotient fl(d / r) by true fp32 division (an
  exact reciprocal multiply when r is a power of two), round-half-even, |q| <= 1 on every axis; the coarsest-level pre-test
  max|d| < cube_threshold(r_coarsest).
* The lookup's 32-NN select: the distance (dx*dx + dy*dy) + dz*dz, each op rounded to fp32; the kernel's own slot order.
* The kNN graph (k_knn, k_knn_grid): the reference's expanded distance, op for op, ranked on (distance, id).

numpy float32 arithmetic is IEEE round-to-nearest and never contracted, so each rule is restated with the ops it names.
Shared by tests/test_host_ties_and_boundaries.py and tests/test_gpu_ties_and_boundaries.py."""
import numpy as np
import torch

F32 = np.float32
KNN = 32


# ------------------------------------------------------------------------------------------------------------------------
# lookup cells
# ------------------------------------------------------------------------------------------------------------------------
def level_scales(base, levels):
    """Cell edge per level: the C entry point takes the base scale as a float, then r = (float)((double)base * 2^l)."""
    b = np.float64(F32(base))
    return [F32(b * 2.0 ** lvl) for lvl in range(levels)]


def is_pow2(r):
    m, _ = np.frexp(np.float64(r))
    return r > 0 and m == 0.5


def cube_threshold(r):
    """The smallest float t with fl(t / r) >= 1.5: max|d| < t  <=>  |rint(fl(d / r))| <= 1 on every axis."""
    r = F32(r)
    t = F32(1.5) * r
    while t / r >= F32(1.5):
        t = np.nextafter(t, F32(0))
    while t / r < F32(1.5):
        t = np.nextafter(t, F32(np.inf))
    return t


def quotient(d, r):
    """fl(d / r) as the kernels form it: a multiply by the exact reciprocal for a power-of-two r, else true division."""
    r = F32(r)
    d = np.asarray(d, dtype=F32)
    return d * (F32(1) / r) if is_pow2(r) else d / r


def cell_codes(d, r):
    """d [..., 3] float32 offsets -> cell in [0, 27) of the 3x3x3 cube at edge r, or -1 outside."""
    q = np.rint(quotient(d, r))
    ok = (np.abs(q) <= 1).all(-1)
    cell = ((q[..., 0] + 1) * 9 + (q[..., 1] + 1) * 3 + (q[..., 2] + 1)).astype(np.int64)
    return np.where(ok, cell, -1)


def offsets(cand, coords):
    """cand [B,N,K,3], coords [B,N,3] (float32) -> fl(cand - coords)."""
    return (np.asarray(cand, F32) - np.asarray(coords, F32)[..., None, :]).astype(F32)


def lookup_cells(cand, coords, base, levels):
    """[B,N,K,levels] int: the cell of every candidate at every level, -1 where the pre-test or the cube rejects it."""
    d = offsets(cand, coords)
    rs = level_scales(base, levels)
    inside = np.abs(d).max(-1) < cube_threshold(rs[-1])
    return np.stack([np.where(inside, cell_codes(d, r), -1) for r in rs], -1)


# ------------------------------------------------------------------------------------------------------------------------
# lookup kNN select
# ------------------------------------------------------------------------------------------------------------------------
def knn_sqdist(cand, coords):
    d = offsets(cand, coords)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def slot_map(k):
    """[32, K/32]: the slot lane `lane` holds as its element e.  A lane streams blocks of VEC consecutive slots, block j at
    j*32*VEC: slot = (e // VEC)*32*VEC + lane*VEC + e % VEC, VEC = min(4, K/32)."""
    kpl = k // 32
    vec = min(4, kpl)
    lane = np.arange(32)[:, None]
    e = np.arange(kpl)[None, :]
    return (e // vec) * 32 * vec + lane * vec + e % vec


def lookup_knn_select(dist):
    """dist [R, K] float32 -> [R, 32] slots in the order k_corr_lookup emits them.  T = the 32nd smallest distance.  If
    exactly 32 candidates are <= T they come in (lane, e) order.  Otherwise (a tie at T) every candidate < T comes first
    in (lane, e) order, then the candidates == T in (lane, e) order up to 32."""
    r, k = dist.shape
    order = slot_map(k).reshape(-1)                  # slots in (lane, e) order
    dl = dist[:, order]
    t = np.sort(dist, -1)[:, KNN - 1:KNN]
    le, lt, eq = dl <= t, dl < t, dl == t
    exact = le.sum(-1, keepdims=True) == KNN
    key = np.where(exact, np.where(le, 0, 2), np.where(lt, 0, np.where(eq, 1, 2)))
    pick = np.argsort(key, -1, kind='stable')[:, :KNN]
    return order[pick]


def lowest_slot_select(dist):
    """The 32 nearest with ties at the 32nd place going to the lowest slots, in ascending slot order."""
    pick = np.lexsort((np.broadcast_to(np.arange(dist.shape[1]), dist.shape), dist), -1)[:, :KNN]
    return np.sort(pick, -1)


# ------------------------------------------------------------------------------------------------------------------------
# kNN graph distance (torch: runs on CPU tensors in the host tests and on the device in the GPU tests)
# ------------------------------------------------------------------------------------------------------------------------
def fma32(a, b, c):
    """Exact fp32 fused multiply-add of float32 tensors.  a*b is exact in double (48 significant bits); s = fl64(a*b + c)
    and its TwoSum error e give the exact sum s + e.  Rounding s to fp32 is right unless s is exactly halfway between two
    floats while e != 0: then the sign of e decides."""
    p = a.double() * b.double()
    cd = c.double()
    s = p + cd
    bb = s - p
    e = (p - (s - bb)) + (cd - bb)
    r = s.float()
    rd = r.double()
    o = torch.nextafter(r, torch.where(s > rd, torch.full_like(r, float('inf')), torch.full_like(r, -float('inf'))))
    od = o.double()
    mid = (s != rd) & (s == (rd + od) * 0.5) & (e != 0)
    toward_o = (e > 0) == (od > rd)
    return torch.where(mid & toward_o, o, r)


def sqnorm32(x):
    """(x*x + y*y) + z*z in fp32 over the last axis."""
    return (x[..., 0] * x[..., 0] + x[..., 1] * x[..., 1]) + x[..., 2] * x[..., 2]


def graph_distance(q, p, mode):
    """q [S,3], p [N,3] float32 -> [S,N]: dot = fma(qz, pz, fma(qy, py, qx*px)); mode 0 (graph.py:53-57) (|q|^2 + |p|^2) - 2 dot,
    mode 1 (pointconv.py:21-24) (-2 dot + |q|^2) + |p|^2."""
    qx, qy, qz = (q[:, i:i + 1].expand(-1, p.shape[0]) for i in range(3))
    px, py, pz = (p[None, :, i].expand(q.shape[0], -1) for i in range(3))
    dot = fma32(qz, pz, fma32(qy, py, qx * px))
    qn, pn = sqnorm32(q)[:, None], sqnorm32(p)[None, :]
    if mode == 0:
        return (qn + pn) - 2.0 * dot
    return (-2.0 * dot + qn) + pn


def knn_graph(xyz, query, k, mode, chunk=1024):
    """xyz [N,3], query [S,3] -> (ids [S,k] int64 in (distance, id) order, rel [S,k,3] = xyz[id] - query)."""
    out = []
    for s0 in range(0, query.shape[0], chunk):
        d = graph_distance(query[s0:s0 + chunk], xyz, mode)
        out.append(torch.sort(d, dim=-1, stable=True).indices[:, :k])
    ids = torch.cat(out)
    return ids, xyz[ids] - query[:, None, :]


# ------------------------------------------------------------------------------------------------------------------------
# boundary-case generators
# ------------------------------------------------------------------------------------------------------------------------
def quotient_boundary(r, h):
    """The smallest positive float d with fl(d / r) >= h."""
    r, h = F32(r), F32(h)
    d = h * r
    while quotient(d, r) >= h:
        d = np.nextafter(d, F32(0))
    while quotient(d, r) < h:
        d = np.nextafter(d, F32(np.inf))
    return d


def boundary_values(base, levels):
    """1-D offsets where a decision flips, both signs: per level the float where fl(d / r) reaches 0.5, passes 0.5 (where
    round-half-even flips: 0.5 itself rounds to 0) and reaches 1.5, its successor and its two predecessors; the pre-test
    threshold, its successor and its predecessor."""
    vals = []
    for r in level_scales(base, levels):
        for h in (0.5, np.nextafter(F32(0.5), F32(1)), 1.5):
            b = quotient_boundary(r, h)
            p = np.nextafter(b, F32(0))
            vals += [b, np.nextafter(b, F32(np.inf)), p, np.nextafter(p, F32(0))]
    t = cube_threshold(level_scales(base, levels)[-1])
    vals += [t, np.nextafter(t, F32(0)), np.nextafter(t, F32(np.inf))]
    v = np.array(vals, F32)
    return np.concatenate([v, -v])


def lattice_pool(base, levels, pool, rng):
    """[pool, 3] distinct offsets on the lattice of step r0/4 within +-3 r_coarsest: every quotient is a multiple of 0.25
    at the finest level (of 2^-l/4 at level l), so +-0.5, +-1.5 and +-2.5 occur at every level."""
    step = np.float64(F32(base)) / 4
    span = int(round(3 * 2 ** (levels - 1) * 4))
    seen, out = set(), []
    while len(out) < pool:
        v = tuple(rng.integers(-span, span + 1, 3).tolist())
        if v not in seen:
            seen.add(v)
            out.append(v)
    return (np.array(out, np.float64) * step).astype(F32)


def boundary_pool(base, levels, pool, rng):
    """[pool, 3] offsets with at least one axis on a value of boundary_values(); the other axes on such a value too
    (probability 1/2 each) or uniform inside the coarsest cube."""
    vals = boundary_values(base, levels)
    t = float(cube_threshold(level_scales(base, levels)[-1]))
    out = rng.uniform(-t, t, (pool, 3)).astype(F32)
    axis = rng.integers(0, 3, pool)
    other = rng.random((pool, 3)) < 0.5
    pick = vals[rng.integers(0, len(vals), (pool, 3))]
    out = np.where(other, pick, out)
    out[np.arange(pool), axis] = vals[rng.integers(0, len(vals), pool)]
    return out


def duplicate_pool(base, levels, pool, rng, dups=40):
    """The query itself `dups` times (distance 0: a tie of 40 at the 32nd place), then lattice offsets."""
    return np.concatenate([np.zeros((dups, 3), F32), lattice_pool(base, levels, pool - dups, rng)])


def cluster_far_pool(pool, rng, near=40):
    """`near` offsets within 1 cm, the rest 10-60 m away: the 32nd distance lies far more than 4 octaves below the largest
    lane minimum, so the select runs its histogram's bucket 0 and a long bisection."""
    a = rng.uniform(-0.01, 0.01, (near, 3))
    u = rng.normal(size=(pool - near, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    far = u * rng.uniform(10.0, 60.0, (pool - near, 1))
    return np.concatenate([a, far]).astype(F32)


POOLS = {'lattice': lattice_pool, 'boundary': boundary_pool, 'duplicate': duplicate_pool}

# query centres: near the origin (sums with the offsets are exact), near 35 and near 1e3 (x - c lands on the coarse grid
# of the centre's ulp)
CENTRES_EXACT = [(0.0, 0.0, 0.0), (0.5, -0.75, 1.25), (-2.0, 1.5, 0.25)]
CENTRES_FAR = [(35.0625, -34.9375, 35.5), (1000.25, -999.5, 1000.75)]


def make_case(kind, base, levels, k, rows, seed, centres=None, pool=None, table_rows=0):
    """A lookup input built from pools of offsets around a few query centres.  Each row's query is a centre; its K
    candidates are a random K-subset of that centre's pool in random slot order (a duplicate / cluster pool's first 40 are
    always included).  Returns dict(xyz2 [1,M,3], idx [1,N,K], coords [1,N,3], val [1,N,K], cand [1,N,K,3], intended
    [1,N,K,3] (centre + offset in float64, to see which candidates hit their intended offset)).  `table_rows` pads the table
    with far points no row uses (to move it out of shared memory)."""
    rng = np.random.default_rng(seed)
    centres = CENTRES_EXACT + CENTRES_FAR if centres is None else centres
    pool = pool or k + max(48, k // 4)
    tabs, offs = [], []
    for c in centres:
        if kind == 'cluster_far':
            o = cluster_far_pool(pool, rng)
        else:
            o = POOLS[kind](base, levels, pool, rng)
        offs.append(o)
        tabs.append((np.asarray(c, F32)[None, :] + o).astype(F32))
    must = min(40, k) if kind in ('duplicate', 'cluster_far') else 0
    tab = np.concatenate(tabs)
    if table_rows > tab.shape[0]:
        tab = np.concatenate([tab, rng.uniform(500, 600, (table_rows - tab.shape[0], 3)).astype(F32)])
    idx = np.empty((rows, k), np.int64)
    coords = np.empty((rows, 3), F32)
    intended = np.empty((rows, k, 3), np.float64)
    for i in range(rows):
        ci = i % len(centres)
        sub = np.concatenate([np.arange(must), must + rng.permutation(pool - must)[:k - must]])
        sub = sub[rng.permutation(k)]
        idx[i] = ci * pool + sub
        coords[i] = np.asarray(centres[ci], F32)
        intended[i] = offs[ci][sub].astype(np.float64)
    val = (rng.normal(20.0, 5.0, (rows, k))).astype(F32)
    cand = tab[idx]
    return dict(xyz2=tab[None], idx=idx[None], coords=coords[None], val=val[None], cand=cand[None], intended=intended[None])


def boundary_classes(cand, coords, intended, base, levels):
    """Counts of the decisions a case reaches: per level, offsets whose quotient is exactly +-0.5 / +-1.5 / +-2.5 (where
    rint and round differ at 0.5, and 1.5 goes outside); offsets on the first float whose quotient reaches 0.5 / 1.5
    ('at') and on the float before it ('below'); offsets exactly at the pre-test threshold or one float either side;
    candidates whose float offset equals the intended one."""
    d = offsets(cand, coords)
    counts = {'exact_offset': int((d.astype(np.float64) == intended).all(-1).sum())}
    a = np.abs(d)
    for lvl, r in enumerate(level_scales(base, levels)):
        q = np.abs(quotient(d, r))
        for h in (0.5, 1.5, 2.5):
            counts[f'l{lvl}_q=={h}'] = int((q == F32(h)).sum())
        for h in (0.5, 1.5):
            b = quotient_boundary(r, h)
            counts[f'l{lvl}_at({h})'] = int((a == b).sum())
            counts[f'l{lvl}_below({h})'] = int((a == np.nextafter(b, F32(0))).sum())
    t = cube_threshold(level_scales(base, levels)[-1])
    a = np.abs(d).max(-1)
    counts['max|d|==thr'] = int((a == t).sum())
    counts['max|d|==prev(thr)'] = int((a == np.nextafter(t, F32(0))).sum())
    counts['max|d|==next(thr)'] = int((a == np.nextafter(t, F32(np.inf))).sum())
    return counts
