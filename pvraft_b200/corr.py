"""CorrBlock -- mirror of the reference module (model/corr.py:8-100): same constructor, parameters,
state_dict keys and call surface (`init_module`, `__call__(coords)`, `get_voxel_feature`,
`get_knn_feature`, `calculate_corr`), with the arithmetic on the H100 kernels.

State layout differs from the reference on purpose: instead of the materialised
`truncate_xyz2 [B,N,K,3]` (12 B/candidate) the block keeps the candidate INDEX (int32) next to the
correlation value -- 8 B per candidate per iteration is the whole HBM stream of the lookup kernel;
xyz is gathered from a 12 B/point table staged in shared memory, and the K candidates of a row are
stored in a bank-aware order (their order carries no meaning in the reference beyond fp summation
order).  `truncated_corr` (sorted, as in the reference) and `truncate_xyz2` stay available as
properties for API parity.
"""
import torch
import torch.nn as nn

from . import ops
from .ops import ACT_LRELU, ACT_NONE, ACT_RELU


def _w(p):
    return p.detach()


def fold_corr_motion(w_cc, b_cc, w_out, b_out, w_kout, b_kout):
    """conv_corr(out_conv.3(a) + knn_out(k)) = W_cc [W_out | W_kout] [a, k] + (W_cc (b_out + b_kout) + b_cc)
    (model/corr.py:45 then model/update.py:16): the folded [64,192] weight and [64] bias, float64 products rounded once."""
    wc = w_cc.detach().reshape(64, 64).double()
    wcat = torch.cat([w_out.detach().reshape(64, 128), w_kout.detach().reshape(64, 64)], 1).double()
    return ((wc @ wcat).float().contiguous(),
            (wc @ (b_out.detach().double() + b_kout.detach().double()) + b_cc.detach().double()).float().contiguous())


class CorrBlock(nn.Module):
    def __init__(self, num_levels=3, base_scale=0.25, resolution=3, truncate_k=128, knn=32):
        super().__init__()
        if resolution != 3:
            raise NotImplementedError('the lookup kernel implements the 3x3x3 cube the reference uses (resolution=3)')
        if knn != ops.KNN:
            raise NotImplementedError('the lookup kernel selects 32 neighbours (model/corr.py:9)')
        self.truncate_k = truncate_k
        self.num_levels = num_levels
        self.resolution = resolution
        self.base_scale = base_scale
        self.out_conv = nn.Sequential(
            nn.Conv1d((self.resolution ** 3) * self.num_levels, 128, 1),
            nn.GroupNorm(8, 128),
            nn.PReLU(),
            nn.Conv1d(128, 64, 1),
        )
        self.knn = knn
        self.knn_conv = nn.Sequential(
            nn.Conv2d(4, 64, 1),
            nn.GroupNorm(8, 64),
            nn.PReLU(),
        )
        self.knn_out = nn.Conv1d(64, 64, 1)
        self.corr_val = None     # [B,N1,K] f32 correlation of the kept candidates (bank-aware order, see ops.corr_reorder)
        self.corr_idx = None     # [B,N1,K] int32 candidate ids (rows of xyz2 [B,N2,3]), same order
        # torch.bfloat16 = the reduced-precision state of BASELINE configs[2] (bf16 values + uint16 ids, 4 B per candidate and
        # iteration; index math stays fp32): inference only, set through RSF.set_precision('bf16')
        self.state_dtype = torch.float32
        self._xyz2 = None
        self._xyz2p = None   # [B,N2,4] (x,y,z,0): the lookup kernel's gather table

    # ------------------------------------------------------------------------------------------
    @staticmethod
    def calculate_corr_pm(fmap1_pm, fmap2_pm):
        """Point-major feature maps [B,N1,C], [B,N2,C] -> corr [B,N1,N2] = <f1_i, f2_j> / sqrt(C) on the wgmma GEMM (3xTF32,
        fp32-accurate).  The kernel works on 128-point tiles: a ragged N1 or N2 is zero-padded to the next multiple of 128 and
        the result cropped (no library GEMM on any path)."""
        b, n, c = fmap1_pm.shape
        if c % 32 != 0:
            raise NotImplementedError(f'calculate_corr: {c} feature channels (the wgmma GEMM needs a multiple of 32; the model has 128)')
        return ops.corr_dense(fmap1_pm, fmap2_pm)

    @staticmethod
    def calculate_corr(fmap1, fmap2):
        """model/corr.py:95-100 with the reference's channel-major [B,C,N] arguments."""
        return CorrBlock.calculate_corr_pm(ops.transpose(fmap1.detach().contiguous().float()),
                                           ops.transpose(fmap2.detach().contiguous().float()))

    def init_module(self, fmap1, fmap2, xyz2):
        """model/corr.py:31-42: build the truncated correlation state for one forward pass
        (fmap1 [B,C,N1], fmap2 [B,C,N2] channel-major as in the reference; xyz2 [B,N2,3])."""
        return self.init_module_pm(ops.transpose(fmap1.detach().contiguous().float()),
                                   ops.transpose(fmap2.detach().contiguous().float()), xyz2)

    def init_module_pm(self, fmap1_pm, fmap2_pm, xyz2):
        """Same with point-major feature maps fmap1 [B,N1,C], fmap2 [B,N2,C] (what the encoders produce natively).  The state
        has N1 rows of K candidates, each a row of xyz2 [B,N2,3]."""
        b, n_p, _ = xyz2.shape
        if fmap2_pm.shape[:2] != (b, n_p) or fmap1_pm.shape[0] != b:
            raise ValueError(f'init_module: fmap1 {tuple(fmap1_pm.shape)}, fmap2 {tuple(fmap2_pm.shape)} and xyz2 {tuple(xyz2.shape)} '
                             'disagree (expected [B,N1,C], [B,N2,C], [B,N2,3])')
        if n_p < self.truncate_k:
            raise ValueError(f'truncate_k={self.truncate_k} exceeds the number of points {n_p}')
        # wgmma GEMM (3xTF32, fp32-accurate) + top-K; in column windows above 49152 points (ops.CorrPlan)
        val, idx = ops.corr_build(fmap1_pm.contiguous(), fmap2_pm.contiguous(), self.truncate_k)
        self._install(*ops.corr_reorder(val, idx), n_p)
        self._xyz2 = xyz2.detach().contiguous().float()
        self._xyz2p = ops.xyz_pad(self._xyz2)

    def set_state(self, truncated_corr, corr_idx, xyz2):
        """Install an externally built state (tests / benchmarks): corr [B,N1,K] f32, idx [B,N1,K] int rows of xyz2 [B,N2,3]."""
        self._install(*ops.corr_reorder(truncated_corr.contiguous().float(), corr_idx.contiguous().to(torch.int32)), xyz2.shape[1])
        self._xyz2 = xyz2.contiguous().float()
        self._xyz2p = ops.xyz_pad(self._xyz2)

    def _install(self, val, idx, n2):
        if self.state_dtype == torch.bfloat16:
            val, idx = ops.corr_state_pack_bf16(val, idx, n2)
        self.corr_val, self.corr_idx = val, idx

    def candidate_ids(self):
        """[B,N,K] int64 rows of xyz2, in the stored order (the uint16 ids of the bf16 state live in an int16 tensor)."""
        if self.corr_idx.dtype == torch.int16:
            return self.corr_idx.to(torch.int32).bitwise_and(0xFFFF).long()
        return self.corr_idx.long()

    @property
    def truncated_corr(self):
        """[B,N,K] correlation values sorted descending, as the reference keeps them (model/corr.py:38)."""
        return None if self.corr_val is None else torch.sort(self.corr_val.float(), dim=2, descending=True).values

    @property
    def truncate_xyz2(self):
        """[B,N,K,3] candidate coordinates, materialised on demand (model/corr.py:42)."""
        b, n, k = self.corr_idx.shape
        idx = self.candidate_ids().reshape(b, n * k, 1).expand(b, n * k, 3)
        return torch.gather(self._xyz2, 1, idx).reshape(b, n, k, 3)

    @property
    def ones_matrix(self):
        return torch.ones_like(self.corr_val, dtype=torch.float32)

    # ------------------------------------------------------------------------------------------
    def lookup(self, coords, **kw):
        """Index + reduce part of the lookup (pvraft_corr_lookup_fwd) -> dict(vox, knn_sel, moments, ...)."""
        if self.corr_val is None:
            raise RuntimeError('CorrBlock.init_module must run before the lookup')
        return ops.corr_lookup(self.corr_val, self.corr_idx, self._xyz2p, coords.detach().contiguous().float(),
                               self.num_levels, self.base_scale, **kw)

    def feature_point_major(self, coords, motion_args=None):
        """coords [B,N,3] -> correlation feature [B,N,64] (point-major).  `motion_args` lets
        UpdateBlock fuse its MotionEncoder into the same launch (see update.py)."""
        b, n, _ = coords.shape
        nvox = self.num_levels * 27
        stats = ops.new_stats(b, coords.device, 1)
        oc, kc = self.out_conv, self.knn_conv
        kpad = (nvox + 31) // 32 * 32
        if ops.tc_supported(n) and kpad - nvox <= 32:
            # out_conv[0] on wgmma: the lookup pads the voxel rows to a multiple of 32 channels (zeros)
            lk = self.lookup(coords, vox_ld=kpad)
            y1 = ops.tc_linear([lk['vox']], ops.tc_weights(oc[0].weight, cols=nvox, k_pad=kpad), _w(oc[0].bias),
                               out_stats=stats[0])
        else:
            lk = self.lookup(coords)
            y1 = ops.linear(lk['vox'], _w(oc[0].weight), _w(oc[0].bias), w_cin=nvox, out_stats=stats[0], out_act=ACT_NONE)
        corr = torch.empty(b, n, 64, dtype=torch.float32, device=coords.device)
        a = ops.pack.CorrFeatArgs(y1=y1, y1_stats=stats[0], gn1_gamma=_w(oc[1].weight), gn1_beta=_w(oc[1].bias),
                                  prelu1=_w(oc[2].weight), w_out=_w(oc[3].weight), b_out=_w(oc[3].bias), knn_sel=lk['knn_sel'],
                                  moments=lk['moments'], w_knn=_w(kc[0].weight), b_knn=_w(kc[0].bias), gnk_gamma=_w(kc[1].weight),
                                  gnk_beta=_w(kc[1].bias), preluk=_w(kc[2].weight), w_kout=_w(self.knn_out.weight),
                                  b_kout=_w(self.knn_out.bias), corr_feat=corr, B=b, N=n)
        keep = [lk, y1, stats, corr]
        if motion_args is not None:
            motion_args(a, keep)
        ops.corr_feature(a)
        return corr, keep

    def feature_motion_tc(self, coords, flow, motion_encoder, need_corr=True):
        """Lookup + feature head + MotionEncoder with every 1x1 convolution on the Hopper tensor cores (wgmma)
        (model/corr.py:42-45 and model/update.py:15-21): coords, flow [B,N,3] -> (corr [B,N,64], motion [B,N,64]);
        with need_corr=False the correlation feature itself is not materialised (one launch fewer) and None is returned.
        Needs ops.tc_supported(N)."""
        y1, kfeat, cflow, gn = self.motion_inputs_tc(coords, flow, motion_encoder)
        oc, me = self.out_conv, motion_encoder
        if need_corr:
            # corr = out_conv[3](PReLU(GN(y1))) + knn_out(kfeat): one GEMM over K = 128 + 64
            bias = ops.derived((oc[3].bias, self.knn_out.bias), 'sum', lambda x, y: (x.detach() + y.detach()).contiguous())
            corr = ops.tc_linear([y1, kfeat], ops.tc_weights((oc[3].weight, self.knn_out.weight), kcat=True), bias, **gn)
            cc = ops.tc_linear([corr], ops.tc_weights(me.conv_corr.weight), _w(me.conv_corr.bias), out_act=ACT_RELU)
        else:
            w_eff, b_eff = self.corr_motion_weights(me)
            corr = None
            cc = ops.tc_linear([y1, kfeat], ops.tc_weights(w_eff), b_eff, out_act=ACT_RELU, **gn)
        motion = ops.tc_linear([cc, cflow], ops.tc_weights(me.conv.weight), _w(me.conv.bias), out_act=ACT_RELU, tail=flow)
        return corr, motion

    def corr_motion_weights(self, motion_encoder):
        """The loop only consumes relu(conv_corr(corr)) (update.py:16), and corr is linear in [a1, kfeat]: conv_corr folded
        into the weights, W_cc [W_out | W_kout] with bias W_cc (b_out + b_kout) + b_cc (float64 products, rounded once)."""
        me, oc = motion_encoder, self.out_conv
        return ops.derived((me.conv_corr.weight, me.conv_corr.bias, oc[3].weight, oc[3].bias, self.knn_out.weight,
                            self.knn_out.bias), 'corr_cc', fold_corr_motion)

    def motion_inputs_tc(self, coords, flow, motion_encoder):
        """The lookup, out_conv[0] and the kNN branch: (y1 [B,N,128] before its GroupNorm, kfeat [B,N,64], cflow [B,N,64],
        the keyword arguments of y1's GroupNorm + PReLU prologue).  Needs ops.tc_supported(N)."""
        b, n, _ = coords.shape
        dev = coords.device
        nvox = self.num_levels * 27
        kpad = (nvox + 31) // 32 * 32
        oc, kc, me = self.out_conv, self.knn_conv, motion_encoder
        stats = ops.new_stats(b, dev, 1)
        lk = self.lookup(coords, vox_ld=kpad)
        y1 = ops.tc_linear([lk['vox']], ops.tc_weights(oc[0].weight, cols=nvox, k_pad=kpad), _w(oc[0].bias), out_stats=stats[0])
        # kNN branch (ALU) + flow embedding
        preluk_host = ops.derived((kc[2].weight,), 'slope', lambda w: float(w.detach().reshape(-1)[0]))
        kfeat = torch.empty(b, n, 64, dtype=torch.float32, device=dev)
        cflow = torch.empty(b, n, 64, dtype=torch.float32, device=dev)
        ops.knn_branch(ops.pack.KnnBranchArgs(knn_sel=lk['knn_sel'], moments=lk['moments'], w_knn=_w(kc[0].weight),
                                              b_knn=_w(kc[0].bias), gnk_gamma=_w(kc[1].weight), gnk_beta=_w(kc[1].bias),
                                              preluk=_w(kc[2].weight), preluk_host=preluk_host, kfeat=kfeat, flow=flow,
                                              cflow=cflow, w_cf=_w(me.conv_flow.weight), b_cf=_w(me.conv_flow.bias), B=b, N=n))
        gn = dict(in_stats=stats[0], in_gamma=_w(oc[1].weight), in_beta=_w(oc[1].bias), in_count=float(n) * 16.0, in_act=ACT_LRELU,
                  in_slope=ops.derived((oc[2].weight,), 'slope', lambda w: float(w.detach().reshape(-1)[0])))
        return y1, kfeat, cflow, gn

    def __call__(self, coords):
        """model/corr.py:44-45 -> [B,64,N]."""
        corr, _ = self.feature_point_major(coords)
        return ops.transpose(corr)

    # the two branches separately, for API parity with the reference (model/corr.py:47,75); each runs
    # the fused kernels and zeroes the other branch by linearity of the final sum.
    def get_voxel_feature(self, coords):
        b, n, _ = coords.shape
        lk = self.lookup(coords)
        stats = ops.new_stats(b, coords.device, 1)
        oc = self.out_conv
        y1 = ops.linear(lk['vox'], _w(oc[0].weight), _w(oc[0].bias), w_cin=self.num_levels * 27, out_stats=stats[0])
        act = ops.gn_act(y1, stats[0], _w(oc[1].weight), _w(oc[1].bias), float(n) * 16, ops.ACT_LRELU,
                         float(oc[2].weight.detach().reshape(-1)[0]))
        return ops.transpose(ops.linear(act, _w(oc[3].weight), _w(oc[3].bias)))

    def get_knn_feature(self, coords):
        return self.__call__(coords) - self.get_voxel_feature(coords)
