"""RSF / RSF_refine -- drop-in mirrors of model/RAFTSceneFlow.py:10-50 and
model/RAFTSceneFlowRefine.py:10-48: same constructor (`args.corr_levels/base_scales/truncate_k`),
same submodule attribute names and state_dict keys, same `forward(p, num_iters)` contract.

The loop body keeps every tensor point-major on the device, launches a fixed sequence of kernels
per iteration with no host synchronisation, and fuses the RAFT glue (flow = coords2 - coords1,
coords2 += delta, model/RAFTSceneFlow.py:41-46) into the first / last kernel of the iteration.
"""
import os

import torch
import torch.nn as nn

from . import ops, train
from .corr import CorrBlock
from .extractor import FlotEncoder
from .graph import Graph
from .refine import FlotRefine
from .update import UpdateBlock


def _records_grad(module):
    """True when the caller differentiates through this forward (tools/engine.py:140-143): the training path of train.py runs;
    otherwise (torch.no_grad(), or nothing requires grad) the fused inference kernels do."""
    if not torch.is_grad_enabled():
        return False
    for m in module.modules():
        # nn.DataParallel replicas keep their (non-leaf) parameter copies in `_former_parameters`; `.parameters()` is empty there
        for t in list(m._parameters.values()) + list(getattr(m, '_former_parameters', {}).values()):
            if t is not None and t.requires_grad:
                return True
    return False


class _RaftBase(nn.Module):
    # CUDA-graph replay of the whole forward (encoders, correlation build, all iterations): the eager path costs ~28 us of
    # host time per launch (python + ctypes + tensor-map encodes), which bounds small batches (B <= 2: ~0.5 ms per
    # iteration) and leaves larger ones exposed to host jitter (at B = 8 the 431 launches of a forward have 45 us each: the
    # same forward measured 19.5 ms on a quiet host and 20.5-21.3 ms next to a busy thread; replayed it is 19.5 ms either
    # way).  `use_cuda_graph = None` (default) replays graphs for inference batches of at most 2 samples from the first call,
    # and for larger batches from the SECOND call with the same shape and unchanged weights (a stream of differently sized
    # clouds, or evaluation calls interleaved with optimizer steps, stays eager: a capture costs three forwards);
    # True / False (or PVRAFT_CUDA_GRAPH=1 / 0) force it on / off.  One graph per (B, N, num_iters), at most 8 kept; inputs are
    # copied into the graph's static buffers, outputs are returned as copies.  The kernels read DERIVED copies of the weights
    # (tf32 hi/lo splits, folded products, bias sums, PReLU slopes known to the host) that are fixed at capture time, so a
    # graph is only valid for the parameter values it was captured with: every entry records (version, data_ptr) of all
    # parameters and is re-captured when any of them changed (optimizer step, load_state_dict, .to()).
    use_cuda_graph = {'1': True, '0': False}.get(os.environ.get('PVRAFT_CUDA_GRAPH', ''), None)

    def reset_graphs(self):
        self.__dict__.pop('_graphs', None)
        self.__dict__.pop('_seen', None)

    def set_precision(self, mode):
        """'fp32' (default): the reference's arithmetic.  'bf16': the reduced-precision STATE mode of BASELINE.json configs[2] --
        the truncated correlation is kept as bf16 values + uint16 candidate ids (4 B instead of 8 B per candidate and iteration,
        the lookup kernel's whole HBM stream); coordinates, index math and every layer stay fp32.  Inference only."""
        if mode not in ('fp32', 'bf16'):
            raise ValueError("precision must be 'fp32' or 'bf16'")
        self.corr_block.state_dtype = torch.bfloat16 if mode == 'bf16' else torch.float32
        self.reset_graphs()
        return self

    def _graph_key(self, xyz1, num_iters):
        # a graph records the kernels of one setting of torch.use_deterministic_algorithms: never replayed under the other
        return (tuple(xyz1.shape), xyz1.device, int(num_iters), ops.deterministic())

    def _stamp(self):
        return tuple((q._version, q.data_ptr()) for q in self.parameters())

    def _graphed(self, p, num_iters):
        xyz1, xyz2 = p[0].detach().contiguous().float(), p[1].detach().contiguous().float()
        graphs = self.__dict__.setdefault('_graphs', {})
        key = self._graph_key(xyz1, num_iters)
        entry = graphs.get(key)
        stamp = self._stamp()
        if entry is not None and entry[3] != stamp:
            entry = None                                   # weights changed since the capture: stale derived constants
        if entry is None:
            static_in = [torch.empty_like(xyz1), torch.empty_like(xyz2)]
            static_in[0].copy_(xyz1)
            static_in[1].copy_(xyz2)
            side = torch.cuda.Stream(device=xyz1.device)   # warm-up off the capture stream: weight splits, derived constants
            side.wait_stream(torch.cuda.current_stream(xyz1.device))
            with torch.cuda.stream(side):
                for _ in range(2):
                    self._forward_impl(static_in, num_iters)
            torch.cuda.current_stream(xyz1.device).wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            l0 = ops.launch_count
            with torch.cuda.graph(graph):
                static_out = self._forward_impl(static_in, num_iters)
            graphs.pop(key, None)
            while len(graphs) >= 8:                        # oldest capture out (its private memory pool goes with it)
                graphs.pop(next(iter(graphs)))
            entry = graphs[key] = (graph, static_in, static_out, stamp, ops.launch_count - l0)
        graph, static_in, static_out, _, n_kernels = entry
        static_in[0].copy_(xyz1)
        static_in[1].copy_(xyz2)
        graph.replay()
        ops.launch_count += n_kernels            # the library's kernels inside the replayed graph
        return static_out.clone() if torch.is_tensor(static_out) else [t.clone() for t in static_out]

    def forward(self, p, num_iters=12):
        if not p[0].is_cuda:
            raise ops._lib.PvraftError('pvraft_b200 kernels need CUDA tensors (no CPU fallback exists)')
        with torch.cuda.device(p[0].device):        # the library launches on the current device
            if _records_grad(self):
                return self._forward_train(p, num_iters)
            graph = self.use_cuda_graph
            if graph is None:    # automatic (never inside an nn.DataParallel replica thread)
                if getattr(self, '_is_replica', False):
                    graph = False
                elif p[0].shape[0] <= 2:
                    graph = True     # host-bound from the first call
                else:                # larger batches: once the same shape has come back with the same weights
                    seen = self.__dict__.setdefault('_seen', {})
                    key, stamp = self._graph_key(p[0], num_iters), self._stamp()
                    graph = seen.get(key) == stamp
                    if len(seen) > 64:
                        seen.clear()
                    seen[key] = stamp
            if graph:
                return self._graphed(p, num_iters)
            return self._forward_impl(p, num_iters)

    def _encode(self, p):
        xyz1, xyz2 = p[0], p[1]
        if xyz1.dim() != 3 or xyz1.shape[-1] != 3 or xyz1.shape != xyz2.shape:
            raise ValueError('expected p = [xyz1 [B,N,3], xyz2 [B,N,3]]')
        xyz1 = xyz1.detach().contiguous().float()
        xyz2 = xyz2.detach().contiguous().float()
        # both clouds go through the shared feature encoder as one batch of 2B samples (RAFTSceneFlow.py:25-26: every op is
        # per sample): half the launches, and 2B*N/128 tiles fill the 132 SMs more evenly
        b = xyz1.shape[0]
        both = torch.cat([xyz1, xyz2], 0)
        fmap, graph2 = self.feature_extractor(both, point_major=True)
        fmap1, fmap2 = fmap[:b], fmap[b:]
        graph = Graph(graph2.nbr[:b], graph2._rel[:b], graph2.k_neighbors, [b * xyz1.shape[1]] * 2,
                      None if graph2.order is None else graph2.order[:b])   # pc1's graph
        self.corr_block.init_module_pm(fmap1, fmap2, xyz2)               # :29
        # the reference rebuilds the same pc1 graph for the context encoder (:31); reuse it
        fct1, graph_context = self.context_extractor(xyz1, graph=graph, point_major=True)
        net = torch.tanh(fct1[..., :self.hidden_dim]).contiguous()       # :33-35 (point-major split)
        inp = torch.relu(fct1[..., self.hidden_dim:]).contiguous()
        return xyz1, xyz2, graph, graph_context, net, inp

    def _iterate(self, xyz1, graph_context, net, inp, num_iters, keep_all):
        b, n, _ = xyz1.shape
        coords2 = xyz1.clone()
        flow = torch.zeros_like(xyz1)
        preds = []
        me = self.update_block.motion_encoder
        use_tc = ops.tc_supported(n)
        # (hoisting the constant context part of the GRU pre-activations out of the loop -- K = 128 per iteration instead of 192 --
        #  was measured slower in round 1, 22.15 vs 21.72 ms per forward: the two extra per-point reads outweigh the shorter GEMM)
        # per iteration: the lookup moments, the lookup-feature GroupNorm sums and the three SetConv sums; one memset
        with ops.stats_arena(b, xyz1.device, 5 * num_iters):
            return self._iterate_body(xyz1, graph_context, net, inp, num_iters, keep_all, coords2, flow, preds, me, use_tc)

    def _iterate_body(self, xyz1, graph_context, net, inp, num_iters, keep_all, coords2, flow, preds, me, use_tc):
        b, n, _ = xyz1.shape
        for _ in range(num_iters):
            if use_tc:
                _, motion = self.corr_block.feature_motion_tc(coords2, flow, me, need_corr=False)          # :42 + update.py:83
            else:
                motion = torch.empty(b, n, 64, dtype=torch.float32, device=xyz1.device)

                def attach(a, keep, flow=flow, motion=motion):
                    me.fill(a, flow)
                    a.motion = ops._p(motion)
                    keep.append(motion)

                _, keep = self.corr_block.feature_point_major(coords2, motion_args=attach)   # :42 + update.py:83
            new_flow = torch.empty_like(xyz1)
            net, _ = self.update_block.forward_pm(net, inp, motion, graph_context, coords1=xyz1, coords2=coords2,
                                                  coords2_out=coords2, flow_out=new_flow)   # :44-46
            flow = new_flow
            if keep_all:
                preds.append(flow)
        return flow, preds


class RSF(_RaftBase):
    def __init__(self, args):
        super().__init__()
        self.hidden_dim = 64
        self.context_dim = 64
        self.feature_extractor = FlotEncoder()
        self.context_extractor = FlotEncoder()
        self.corr_block = CorrBlock(num_levels=args.corr_levels, base_scale=args.base_scales,
                                    resolution=3, truncate_k=args.truncate_k)
        self.update_block = UpdateBlock(hidden_dim=self.hidden_dim)

    def _forward_impl(self, p, num_iters=12):
        xyz1, _, _, graph_context, net, inp = self._encode(p)
        _, preds = self._iterate(xyz1, graph_context, net, inp, num_iters, keep_all=True)
        return preds

    def _forward_train(self, p, num_iters=12):
        return train.rsf_forward(self, p, num_iters)


class RSF_refine(_RaftBase):
    def __init__(self, args):
        super().__init__()
        self.hidden_dim = 64
        self.context_dim = 64
        self.feature_extractor = FlotEncoder()
        self.context_extractor = FlotEncoder()
        self.corr_block = CorrBlock(num_levels=args.corr_levels, base_scale=args.base_scales,
                                    resolution=3, truncate_k=args.truncate_k)
        self.update_block = UpdateBlock(hidden_dim=self.hidden_dim)
        self.refine_block = FlotRefine()

    def _forward_impl(self, p, num_iters=12):
        xyz1, _, graph, graph_context, net, inp = self._encode(p)
        flow, _ = self._iterate(xyz1, graph_context, net, inp, num_iters, keep_all=False)
        return self.refine_block(flow, graph)      # RAFTSceneFlowRefine.py:46

    def _forward_train(self, p, num_iters=12):
        """model/RAFTSceneFlowRefine.py:22-48: everything up to the last flow under no_grad (the fused inference kernels),
        the refiner -- the only part tools/engine_refine.py trains -- layer by layer with gradients."""
        with torch.no_grad():
            xyz1, _, graph, graph_context, net, inp = self._encode(p)
            flow, _ = self._iterate(xyz1, graph_context, net, inp, num_iters, keep_all=False)
        return train.flot_refine(self.refine_block, flow, graph)
