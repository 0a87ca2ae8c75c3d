"""Generate tests/golden/unequal_rsf.npz: the unmodified reference modules on pairs of clouds of different sizes, on CPU.

    PVRAFT_REFERENCE=<reference tree> python tests/golden/make_golden_unequal.py

CorrBlock.init_module (model/corr.py:31-42) reshapes the top-K indices with the size of xyz2, but their rows belong to
fmap1, so it raises for N1 != N2.  This script builds that state itself with N1 rows -- the reference's own calculate_corr,
torch.topk over the N2 columns, the K candidate rows of xyz2 gathered for each of the N1 rows -- and installs it in place of
init_module; everything downstream is the reference's modules, unchanged, traced by make_golden.trace_forward.

RSF_refine with torch.manual_seed(0) default init and make_golden.randomise_affine(model, 13).  To keep the file small:
  * weights: only the 1-D parameters (biases, GroupNorm and PReLU, which randomise_affine draws) are stored, as 'w/<name>';
    the rest is the default init of seed 0 (conftest.default_weights), pinned by 'wsum' (float64 sum of every tensor, in
    the order of 'wnames');
  * per case: both clouds, the flow of every iteration, and the corr / voxel_feature / net outputs of the first S points
    (they depend on all points, through the GroupNorms and the graph, so the slice is as strict a golden for those points);
  * case c also keeps the truncated state (values + candidate ids into pc2, the reference's order), the query coordinates
    of iteration 1 and their index goldens (cell ids, validity, kNN slots); case a the refined flow; every case the
    checksum of its truncated values (sum, sum of magnitudes).
Cases: a (N1, N2) = (256, 384), B = 2, K = 64; b (384, 256), B = 2, K = 64 (the tensor-core path of the CUDA model);
c (100, 300), B = 1, K = 128 (CUDA-core path) on a compact cloud: every candidate lies within 0.4 of the query, so at the
coarsest level (cell edge 1.0) the central cell counts more than N1 = 100 candidates and clamp(count, 1, N1) is reached.
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as G   # noqa: E402

ITERS, S = 2, 16
CASES = dict(a=(2, 256, 384, 64, 21, 10.0), b=(2, 384, 256, 64, 22, 10.0), c=(1, 100, 300, 128, 23, 0.4))


def init_unequal(cb, fmap1, fmap2, xyz2):
    b, n1, k = fmap1.shape[0], fmap1.shape[2], cb.truncate_k
    top = torch.topk(type(cb).calculate_corr(fmap1, fmap2), k=k, dim=2, sorted=True)
    cb.truncated_corr = top.values
    cb.ones_matrix = torch.ones_like(top.values)
    cb.truncate_xyz2 = torch.gather(xyz2.unsqueeze(1).expand(b, n1, xyz2.shape[1], 3), 2,
                                    top.indices.unsqueeze(-1).expand(b, n1, k, 3))
    cb.golden_indices = top.indices


def main():
    if not G.REF or not os.path.isdir(G.REF):
        sys.exit('set PVRAFT_REFERENCE to the reference tree (weiyithu/PV-RAFT)')
    G.install_scatter_shim()
    sys.path.insert(0, G.REF)
    from model.RAFTSceneFlowRefine import RSF_refine
    torch.set_num_threads(8)
    torch.manual_seed(0)
    model = RSF_refine(types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=64)).eval()
    G.randomise_affine(model, 13)
    sd = model.state_dict()
    names = sorted(sd)
    out = {'w/' + k: v.numpy() for k, v in sd.items() if v.dim() == 1}
    out['wnames'] = np.array(names)
    out['wsum'] = np.array([sd[k].double().sum().item() for k in names])
    out['base_scale'] = np.float32(0.25)
    cb = model.corr_block
    cb.init_module = types.MethodType(init_unequal, cb)   # instead of the class's init_module, inside trace_forward
    for case, (b, n1, n2, k, seed, scale) in CASES.items():
        g = torch.Generator().manual_seed(seed)
        pc1 = scale * torch.rand(b, n1, 3, generator=g)
        pc2 = scale * torch.rand(b, n2, 3, generator=g)
        if scale == 10.0:   # a displaced copy of pc1's region, as the synthetic workload, with its own point count
            pc2 = torch.cat([pc1, pc1[:, :max(0, n2 - n1)]], 1)[:, :n2] + 0.1 * torch.randn(b, n2, 3, generator=g)
        cb.truncate_k = k
        tr = G.trace_forward(model, pc1, pc2, ITERS)
        p = case + '/'
        out[p + 'pc1'], out[p + 'pc2'] = pc1.numpy(), pc2.numpy()
        out[p + 'meta'] = np.array([b, n1, n2, k, 3, ITERS, S], dtype=np.int64)
        for it in range(ITERS):
            out[p + f'it{it}/flow'] = tr[f'it{it}/flow']
            for key in ('corr', 'voxel_feature', 'net'):
                out[p + f'it{it}/{key}'] = np.ascontiguousarray(tr[f'it{it}/{key}'][:, :, :S])
        out[p + 'truncated_corr_checksum'] = np.array([tr['truncated_corr'].astype(np.float64).sum(),
                                                      np.abs(tr['truncated_corr']).astype(np.float64).sum()])
        if case == 'c':
            out[p + 'truncated_corr'] = tr['truncated_corr']
            out[p + 'cand'] = cb.golden_indices.numpy().astype(np.int16)
            out[p + 'it1/coords'] = tr['it1/coords']
            for lvl in range(3):
                out[p + f'it1/cube_idx_l{lvl}'] = tr[f'it1/cube_idx_l{lvl}']
                out[p + f'it1/valid_l{lvl}'] = tr[f'it1/valid_l{lvl}']
            out[p + 'it1/knn_slots'] = tr['it1/knn_slots']
        if case == 'a':
            with torch.no_grad():
                _, graph = model.feature_extractor(pc1)
                out[p + 'refined'] = model.refine_block(torch.from_numpy(tr[f'it{ITERS - 1}/flow']), graph).numpy()
    path = os.path.join(HERE, 'unequal_rsf.npz')
    np.savez_compressed(path, **out)
    print('unequal_rsf.npz', os.path.getsize(path) // 1024, 'KiB')


if __name__ == '__main__':
    main()
