"""The CPU oracle (oracle/pvraft_oracle.py) extended to pairs of clouds of different sizes, xyz1 [B,N1,3] and xyz2 [B,N2,3].

Only the correlation initialisation depends on the two sizes: its state has N1 rows of K candidates, each a row of xyz2
(model/corr.py:39 reshapes the top-K indices with the size of xyz2, which is right only for N1 == N2; the rows belong to
fmap1).  Everything after it -- the lookup, the update block, the refiner -- is written per cloud, and the oracle's
functions are used unchanged; `voxel_means` already divides by clamp(count, 1, N1), N1 being the size of the query cloud.
`voxel_means` here is the same restatement in the state's own dtype, for float64 gradient references.
"""
import types
from typing import List

import torch

from conftest import default_weights
from oracle import pvraft_oracle as O


def corr_init(fmap1: torch.Tensor, fmap2: torch.Tensor, xyz2: torch.Tensor, truncate_k: int) -> O.CorrState:
    """model/corr.py:31-42 with N1 rows: fmap1 [B,C,N1], fmap2 [B,C,N2], xyz2 [B,N2,3] -> state [B,N1,K(,3)]."""
    b, m, _ = xyz2.shape
    n = fmap1.shape[2]
    top = torch.topk(O.calculate_corr(fmap1, fmap2), k=truncate_k, dim=2, sorted=True)
    cand = torch.gather(xyz2.unsqueeze(1).expand(b, n, m, 3), 2, top.indices.unsqueeze(-1).expand(b, n, truncate_k, 3))
    return O.CorrState(top.values, top.indices, cand)


def prepare(P, xyz1: torch.Tensor, xyz2: torch.Tensor, truncate_k: int) -> O.LoopInputs:
    """O.prepare (model/RAFTSceneFlow.py:24-35) for clouds of different sizes."""
    fmap1, g1 = O.flot_encoder(P, 'feature_extractor', xyz1)
    fmap2, _ = O.flot_encoder(P, 'feature_extractor', xyz2)
    state = corr_init(fmap1, fmap2, xyz2, truncate_k)
    fct1, gctx = O.flot_encoder(P, 'context_extractor', xyz1)
    net, inp = torch.split(fct1, [64, 64], dim=1)
    return O.LoopInputs(state, torch.tanh(net), torch.relu(inp), gctx, g1)


def rsf_forward(P, xyz1, xyz2, num_iters, num_levels=3, base_scale=0.25, truncate_k=512) -> List[torch.Tensor]:
    """O.rsf_forward (model/RAFTSceneFlow.py:22-50) for clouds of different sizes -> flows [B,N1,3]."""
    return O.raft_loop(P, prepare(P, xyz1, xyz2, truncate_k), xyz1, num_iters, num_levels, base_scale)


def voxel_means(state: O.CorrState, coords: torch.Tensor, num_levels: int, base_scale: float) -> torch.Tensor:
    """O.voxel_means (model/corr.py:47-71) accumulated in the dtype of the state's values."""
    b, n, _ = coords.shape
    feats = []
    for lvl in range(num_levels):
        cube, valid = O.voxel_cube_index(state, coords, base_scale * (2 ** lvl))
        w = valid.to(state.truncated_corr.dtype)
        s = torch.zeros(b, n, 27, dtype=w.dtype).scatter_add_(2, cube, state.truncated_corr * w)
        c = torch.zeros(b, n, 27, dtype=w.dtype).scatter_add_(2, cube, w)
        feats.append((s / torch.clamp(c, 1, n)).transpose(1, 2))
    return torch.cat(feats, dim=1).contiguous()


def golden_weights(arr, W1):
    """The golden model's weights: seed-0 default init with the stored 1-D parameters, checked against the stored sums."""
    W = default_weights(refine=True, seed=0, args=types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=64))
    assert set(W1) <= set(W)
    W.update(W1)
    names = [str(n) for n in arr['wnames']]
    assert sorted(W) == names
    sums = torch.tensor([W[n].double().sum().item() for n in names], dtype=torch.float64)
    assert torch.equal(sums, arr['wsum']), 'the default init of seed 0 is not the golden model'
    return W


def golden_state(g):
    """The truncated state stored in unequal_rsf.npz (g: key -> array of one case): values and xyz2 rows of the candidates,
    in the reference's order."""
    idx = g('cand').long()
    pc2 = g('pc2')
    b, n, k = idx.shape
    cand = torch.gather(pc2.unsqueeze(1).expand(b, n, pc2.shape[1], 3), 2, idx.unsqueeze(-1).expand(b, n, k, 3))
    return O.CorrState(g('truncated_corr'), idx, cand)
