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


def _records_grad(module, p):
    """True when the caller differentiates through this forward (tools/engine.py:140-143), w.r.t. a parameter or an input
    cloud of p: the training path of train.py runs; otherwise (torch.no_grad(), or nothing requires grad) the fused
    inference kernels do."""
    if not torch.is_grad_enabled():
        return False
    if p[0].requires_grad or p[1].requires_grad:   # (inside an nn.DataParallel replica: the scattered inputs keep requires_grad)
        return True
    for m in module.modules():
        # nn.DataParallel replicas keep their (non-leaf) parameter copies in `_former_parameters`; `.parameters()` is empty there
        for t in list(m._parameters.values()) + list(getattr(m, '_former_parameters', {}).values()):
            if t is not None and t.requires_grad:
                return True
    return False


def _check_flow_init(p, flow_init):
    """flow_init of forward(): None, or a tensor [B,N1,3] -> its detached, contiguous fp32 form (a constant: RAFT's warm start
    passes no gradient to it)."""
    if flow_init is None:
        return None
    want = (int(p[0].shape[0]), int(p[0].shape[1]), 3) if p[0].dim() == 3 else None
    if not torch.is_tensor(flow_init) or want is None or tuple(flow_init.shape) != want:
        got = tuple(flow_init.shape) if torch.is_tensor(flow_init) else type(flow_init).__name__
        raise ValueError(f'flow_init must be a tensor [B,N1,3] = {want} shaped like the first cloud, got {got}')
    if not flow_init.is_floating_point():
        raise ValueError(f'flow_init must be a floating-point tensor, got {flow_init.dtype}')
    if not flow_init.is_cuda:
        raise ops._lib.PvraftError('pvraft_b200 kernels need CUDA tensors (no CPU fallback exists): flow_init is on the CPU')
    return flow_init.detach().contiguous().float()


def _clone(out):
    """A copy of a graph's static output: a tensor, a list of tensors, or the (forward, backward) pair of either."""
    if torch.is_tensor(out):
        return out.clone()
    return type(out)(_clone(t) for t in out) if isinstance(out, tuple) else [_clone(t) for t in out]


class _RaftBase(nn.Module):
    # CUDA-graph replay of the whole forward (encoders, correlation build, all iterations): the eager path costs ~28 us of
    # host time per launch (python + ctypes + tensor-map encodes), which bounds small batches (B <= 2: ~0.5 ms per
    # iteration) and leaves larger ones exposed to host jitter (at B = 8 the 431 launches of a forward have 45 us each: the
    # same forward measured 19.5 ms on a quiet host and 20.5-21.3 ms next to a busy thread; replayed it is 19.5 ms either
    # way).  `use_cuda_graph = None` (default) replays graphs for inference batches of at most 2 samples from the first call,
    # and for larger batches from the SECOND call with the same shape and unchanged weights (a stream of differently sized
    # clouds, or evaluation calls interleaved with optimizer steps, stays eager: a capture costs three forwards);
    # True / False (or PVRAFT_CUDA_GRAPH=1 / 0) force it on / off.  One graph per (B, N1, N2, num_iters), at most 8 kept; inputs are
    # copied into the graph's static buffers, outputs are returned as copies.  The kernels read DERIVED copies of the weights
    # (tf32 hi/lo splits, folded products, bias sums, PReLU slopes known to the host) that are fixed at capture time, so a
    # graph is only valid for the parameter values it was captured with: every entry records (version, data_ptr) of all
    # parameters and is re-captured when any of them changed (optimizer step, load_state_dict, .to()).
    use_cuda_graph = {'1': True, '0': False}.get(os.environ.get('PVRAFT_CUDA_GRAPH', ''), None)
    bf16_compute = False   # set_precision('bf16-compute' / 'bf16-mixed'): the RAFT loop's tensor-core layers on bf16 operands

    def reset_graphs(self):
        for name in ('_graphs', '_seen', '_stream_graphs', '_stream_seen'):   # (the last two: SceneFlowStream's)
            self.__dict__.pop(name, None)

    def set_precision(self, mode):
        """'fp32' (default): the reference's arithmetic.  'bf16': the reduced-precision STATE mode of BASELINE.json configs[2] --
        the truncated correlation is kept as bf16 values + uint16 candidate ids (4 B instead of 8 B per candidate and iteration,
        the lookup kernel's whole HBM stream); coordinates, index math and every layer stay fp32.  'bf16-compute': the bf16
        state, and every tensor-core layer of the RAFT loop (out_conv[0], the update chain or its five layers, the flow
        head's SetConv fc2 / fc3 and its FLOW layer) on bf16 operands -- activations after the prologue and weights rounded to
        nearest even -- with fp32 accumulation; prologues, epilogues, GroupNorm statistics, coordinates and every tensor in
        memory stay fp32.  The encoders, the correlation build and the refiner stay fp32, so everything before the loop is
        bitwise that of 'bf16'; at N % 128 != 0 the loop runs on the CUDA-core kernels and the mode equals 'bf16'.  Both bf16
        modes are inference only (RSF_refine trains its fp32 refiner behind the no-grad loop).
        'bf16-mixed': mixed-precision training.  The correlation state stays fp32 and the loop's tensor-core layers run on
        bf16 operands with fp32 accumulation, in inference as in 'bf16-compute' and in a training step too: there every
        per-point layer of the loop whose shape suits the tensor cores (train.bf16_layer_plan) takes bf16 wgmma for its
        output, its input gradient and its weight gradient.  The weights stay fp32 (the optimizer's master copy); the
        encoders, the correlation build and lookup, GroupNorm, the edge-level layers, the loss and the refiner keep their
        fp32 forms, so everything before the loop is bitwise 'fp32'.  Input gradients work; at N % 128 != 0 nothing runs on
        the tensor cores and the mode equals 'fp32'."""
        if mode not in ('fp32', 'bf16', 'bf16-compute', 'bf16-mixed'):
            raise ValueError("precision must be 'fp32', 'bf16', 'bf16-compute' or 'bf16-mixed'")
        self.corr_block.state_dtype = torch.float32 if mode in ('fp32', 'bf16-mixed') else torch.bfloat16
        self.bf16_compute = mode in ('bf16-compute', 'bf16-mixed')   # (in __dict__: nn.DataParallel replicas inherit it)
        self.reset_graphs()
        return self

    def _graph_key(self, xyz1, xyz2, num_iters, warm=False, bidirectional=False):
        # a graph records the kernels of one setting of torch.use_deterministic_algorithms: never replayed under the other.
        # A pair of clouds of different sizes adds the second cloud's shape (pairs that share N1 and differ in N2 run on
        # different buffers); a pair of equal sizes keeps the short key.  A warm-started forward (flow_init) records only
        # that it is one: the starting flow is a static input like the clouds, so new values replay the same graph.  A
        # bidirectional forward records its flag.
        key = (tuple(xyz1.shape), xyz1.device, int(num_iters), ops.deterministic())
        key = key if xyz2.shape == xyz1.shape else key + (tuple(xyz2.shape),)
        key = key + ('flow_init',) if warm else key
        return key + ('bidirectional',) if bidirectional else key

    def _stamp(self):
        return tuple((q._version, q.data_ptr()) for q in self.parameters())

    def _graphed(self, p, num_iters, flow_init=None, bidirectional=False):
        xyz1, xyz2 = p[0].detach().contiguous().float(), p[1].detach().contiguous().float()
        inputs = [xyz1, xyz2] if flow_init is None else [xyz1, xyz2, flow_init]
        graphs = self.__dict__.setdefault('_graphs', {})
        key = self._graph_key(xyz1, xyz2, num_iters, flow_init is not None, bidirectional)
        entry = graphs.get(key)
        stamp = self._stamp()
        if entry is not None and entry[3] != stamp:
            entry = None                                   # weights changed since the capture: stale derived constants
        if entry is None:
            static_in = [torch.empty_like(t) for t in inputs]
            for s, t in zip(static_in, inputs):
                s.copy_(t)

            def run():
                return self._forward_impl(static_in[:2], num_iters, static_in[2] if len(static_in) > 2 else None, bidirectional)

            side = torch.cuda.Stream(device=xyz1.device)   # warm-up off the capture stream: weight splits, derived constants
            side.wait_stream(torch.cuda.current_stream(xyz1.device))
            with torch.cuda.stream(side):
                for _ in range(2):
                    run()
            torch.cuda.current_stream(xyz1.device).wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            l0 = ops.launch_count
            with torch.cuda.graph(graph):
                static_out = run()
            graphs.pop(key, None)
            while len(graphs) >= 8:                        # oldest capture out (its private memory pool goes with it)
                graphs.pop(next(iter(graphs)))
            entry = graphs[key] = (graph, static_in, static_out, stamp, ops.launch_count - l0)
        graph, static_in, static_out, _, n_kernels = entry
        for s, t in zip(static_in, inputs):
            s.copy_(t)
        graph.replay()
        ops.launch_count += n_kernels            # the library's kernels inside the replayed graph
        return _clone(static_out)

    def forward(self, p, num_iters=12, flow_init=None, bidirectional=False):
        """p = [xyz1 [B,N1,3], xyz2 [B,N2,3]] -> the reference's outputs.  flow_init [B,N1,3] (optional): RAFT's warm start,
        the loop starts at coords2 = xyz1 + flow_init instead of xyz1.  It is a constant: detached, it receives no gradient.
        None runs the reference's loop; a zero flow_init gives the same bits.
        bidirectional=True: the flow in both directions, (forward, backward) = (model(p), model([xyz2, xyz1])) in one call
        (_encode_both): for RSF two lists of num_iters flows [B,N1,3] and [B,N2,3], for RSF_refine the two refined flows.
        Under torch.use_deterministic_algorithms(True) each equals its one-direction call bitwise when N1 = N2 is a multiple
        of 128 or N1 != N2.  It cannot be warm-started: flow_init must be None."""
        if bidirectional:
            if flow_init is not None:
                raise ValueError('a bidirectional forward cannot be warm-started: flow_init must be None')
            ops.check_pair(p[0], p[1], self.corr_block.truncate_k)   # both directions, before any launch
            ops.check_pair(p[1], p[0], self.corr_block.truncate_k)
            if self.corr_block.state_dtype != torch.float32 and max(p[0].shape[1], p[1].shape[1]) > 65536:
                raise ValueError(f'uint16 candidate ids need both clouds of a bidirectional forward to have at most 65536 points, '
                                 f'got N1={p[0].shape[1]} and N2={p[1].shape[1]}')
        flow_init = _check_flow_init(p, flow_init)
        if not p[0].is_cuda:
            raise ops._lib.PvraftError('pvraft_b200 kernels need CUDA tensors (no CPU fallback exists)')
        with torch.cuda.device(p[0].device):        # the library launches on the current device
            if flow_init is not None and flow_init.device != p[0].device:
                raise ops._lib.PvraftError(f'flow_init is on {flow_init.device}, the clouds on {p[0].device}')
            if _records_grad(self, p):
                return self._forward_train(p, num_iters, flow_init, bidirectional)
            graph = self.use_cuda_graph
            if graph is None:    # automatic (never inside an nn.DataParallel replica thread)
                if getattr(self, '_is_replica', False):
                    graph = False
                elif p[0].shape[0] <= 2:
                    graph = True     # host-bound from the first call
                else:                # larger batches: once the same shape has come back with the same weights
                    seen = self.__dict__.setdefault('_seen', {})
                    key, stamp = self._graph_key(p[0], p[1], num_iters, flow_init is not None, bidirectional), self._stamp()
                    graph = seen.get(key) == stamp
                    if len(seen) > 64:
                        seen.clear()
                    seen[key] = stamp
            if graph:
                return self._graphed(p, num_iters, flow_init, bidirectional)
            return self._forward_impl(p, num_iters, flow_init, bidirectional)

    def _forward_impl(self, p, num_iters=12, flow_init=None, bidirectional=False):
        if not bidirectional:
            return self._run(self._encode(p), num_iters, flow_init)
        outs = [self._run(e, num_iters) for e in self._encode_both(p)]
        if len(outs) == 2:
            return tuple(outs)
        out, b = outs[0], int(p[0].shape[0])
        if torch.is_tensor(out):
            return out[:b], out[b:]
        return [f[:b] for f in out], [f[b:] for f in out]

    def _encode_both(self, p):
        """Yields _pair's outputs for both directions (forward has checked both); the caller runs each before taking the
        next, because _pair leaves the correlation state on corr_block.  Clouds of equal sizes: one 2B stack (xyz1 =
        cat[x1, x2] against cat[x2, x1]) on the encoder's 2B pass, whose graph is kept whole -- each cloud's own graph, for
        the context encoder, the loop's SetConv and the refiner -- so one correlation build, one context pass and one loop
        serve both directions.  Different sizes: each cloud encoded once, then one _pair per direction."""
        xyz1 = p[0].detach().contiguous().float()
        xyz2 = p[1].detach().contiguous().float()
        if xyz1.shape == xyz2.shape:
            b = xyz1.shape[0]
            both = torch.cat([xyz1, xyz2], 0)
            fmap, graph = self.feature_extractor(both, point_major=True)
            yield self._pair(both, torch.cat([xyz2, xyz1], 0), fmap, graph, torch.cat([fmap[b:], fmap[:b]], 0))
            return
        fmap1, graph1 = self._encode_cloud(xyz1)
        fmap2, graph2 = self._encode_cloud(xyz2)
        yield self._pair(xyz1, xyz2, fmap1, graph1, fmap2)
        yield self._pair(xyz2, xyz1, fmap2, graph2, fmap1)

    def _encode(self, p):
        xyz1, xyz2 = p[0], p[1]
        ops.check_pair(xyz1, xyz2, self.corr_block.truncate_k)
        xyz1 = xyz1.detach().contiguous().float()
        xyz2 = xyz2.detach().contiguous().float()
        b = xyz1.shape[0]
        if xyz1.shape == xyz2.shape:
            # both clouds go through the shared feature encoder as one batch of 2B samples (RAFTSceneFlow.py:25-26: every op
            # is per sample): half the launches, and 2B*N/128 tiles fill the 132 SMs more evenly
            both = torch.cat([xyz1, xyz2], 0)
            fmap, graph2 = self.feature_extractor(both, point_major=True)
            fmap1, fmap2 = fmap[:b], fmap[b:]
            graph = Graph(graph2.nbr[:b], graph2._rel[:b], graph2.k_neighbors, [b * xyz1.shape[1]] * 2,
                          None if graph2.order is None else graph2.order[:b])   # pc1's graph
        else:
            # clouds of different sizes: one encoder pass per cloud (the kernels take one N per launch)
            fmap1, graph = self._encode_cloud(xyz1)                     # pc1's graph
            fmap2, _ = self._encode_cloud(xyz2)
        return self._pair(xyz1, xyz2, fmap1, graph, fmap2)

    def _encode_cloud(self, xyz):
        """The part of the pre-loop work that sees one cloud alone: its feature map [B,N,128] and its kNN graph (with the
        Morton order).  Nothing in it depends on which side of a pair the cloud is on, so a scan sequence encodes every scan
        once (SceneFlowStream)."""
        return self.feature_extractor(xyz, point_major=True)

    def _pair(self, xyz1, xyz2, fmap1, graph, fmap2):
        """The pre-loop work that needs both clouds, from their feature maps and pc1's graph -> the loop's inputs."""
        self.corr_block.init_module_pm(fmap1, fmap2, xyz2)               # :29
        # the reference rebuilds the same pc1 graph for the context encoder (:31); reuse it
        fct1, graph_context = self.context_extractor(xyz1, graph=graph, point_major=True)
        net = torch.tanh(fct1[..., :self.hidden_dim]).contiguous()       # :33-35 (point-major split)
        inp = torch.relu(fct1[..., self.hidden_dim:]).contiguous()
        return xyz1, xyz2, graph, graph_context, net, inp

    def _iterate(self, xyz1, graph_context, net, inp, num_iters, keep_all, flow_init=None):
        b, n, _ = xyz1.shape
        if flow_init is None:
            coords2 = xyz1.clone()
            flow = torch.zeros_like(xyz1)
        else:                                     # warm start: the loop starts at xyz1 + flow_init
            coords2 = xyz1 + flow_init
            flow = coords2 - xyz1                 # the first iteration's flow input, as :43 computes it
        preds = []
        me = self.update_block.motion_encoder
        use_tc = ops.tc_supported(n)
        # (hoisting the constant context part of the GRU pre-activations out of the loop -- K = 128 per iteration instead of 192 --
        #  was measured slower in round 1, 22.15 vs 21.72 ms per forward: the two extra per-point reads outweigh the shorter GEMM)
        # per iteration: the lookup moments, the lookup-feature GroupNorm sums and the three SetConv sums; one memset.
        # 'bf16-compute': the loop's tensor-core layers take the bf16 form of their weights (ops.bf16_compute)
        with ops.stats_arena(b, xyz1.device, 5 * num_iters), ops.bf16_compute(self.bf16_compute):
            return self._iterate_body(xyz1, graph_context, net, inp, num_iters, keep_all, coords2, flow, preds, me, use_tc)

    def _iterate_body(self, xyz1, graph_context, net, inp, num_iters, keep_all, coords2, flow, preds, me, use_tc):
        b, n, _ = xyz1.shape
        for _ in range(num_iters):
            if use_tc and ops.fuse_update_chain:
                y1, kfeat, cflow, gn = self.corr_block.motion_inputs_tc(coords2, flow, me)                # :42
                new_flow = torch.empty_like(xyz1)
                net, _ = self.update_block.forward_chain_pm(net, inp, y1, kfeat, cflow, flow, gn,
                                                            self.corr_block.corr_motion_weights(me), graph_context,
                                                            coords1=xyz1, coords2=coords2, coords2_out=coords2,
                                                            flow_out=new_flow)                              # :43-46
                flow = new_flow
                if keep_all:
                    preds.append(flow)
                continue
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

    def _run(self, encoded, num_iters, flow_init=None):
        """The loop on _pair's outputs -> the list of num_iters flows."""
        xyz1, _, _, graph_context, net, inp = encoded
        _, preds = self._iterate(xyz1, graph_context, net, inp, num_iters, keep_all=True, flow_init=flow_init)
        return preds

    def _forward_train(self, p, num_iters=12, flow_init=None, bidirectional=False):
        return train.rsf_forward(self, p, num_iters, flow_init, bidirectional)


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

    def _run(self, encoded, num_iters, flow_init=None):
        """The loop and the refiner on _pair's outputs -> the refined flow."""
        xyz1, _, graph, graph_context, net, inp = encoded
        flow, _ = self._iterate(xyz1, graph_context, net, inp, num_iters, keep_all=False, flow_init=flow_init)
        return self.refine_block(flow, graph)      # RAFTSceneFlowRefine.py:46

    def _forward_train(self, p, num_iters=12, flow_init=None, bidirectional=False):
        """model/RAFTSceneFlowRefine.py:22-48: everything up to the last flow under no_grad (the fused inference kernels),
        the refiner -- the only part tools/engine_refine.py trains -- layer by layer with gradients.  The refiner's input
        flow is coords2 - xyz1 with coords2 computed under no_grad, so xyz1 receives minus the flow's gradient and xyz2 none.
        Bidirectional: the same per direction (the refiner on the 2B stack when the sizes are equal); each cloud receives
        minus the gradient of the refiner input flow that starts on it."""
        starts = (p[0], p[1]) if bidirectional else (p[0],)       # the clouds the refiner's input flows start on
        if any(x.requires_grad for x in starts) and self.corr_block.state_dtype != torch.float32:
            raise NotImplementedError("training differentiates through the fp32 state: call model.set_precision('fp32')")
        with torch.no_grad():
            encoded = self._encode_both(p) if bidirectional else [self._encode(p)]   # (each direction's loop runs before the next _pair)
            loops = [(e[0], e[2], self._iterate(e[0], e[3], e[4], e[5], num_iters, keep_all=False, flow_init=flow_init)[0])
                     for e in encoded]
        if not bidirectional:
            x1 = p[0].float()
            flow, graph = loops[0][2], loops[0][1]
            if x1.requires_grad:
                flow = flow + (x1.detach() - x1)      # the same values; d xyz1 = -d flow
            return train.flot_refine(self.refine_block, flow, graph)
        x1, x2 = p[0].float(), p[1].float()
        if len(loops) == 1:                           # the 2B stack: cat[x1, x2] starts the flows
            b = int(p[0].shape[0])
            start = torch.cat([x1, x2], 0)
            flow = loops[0][2]
            if start.requires_grad:
                flow = flow + (start.detach() - start)
            out = train.flot_refine(self.refine_block, flow, loops[0][1])
            return out[:b], out[b:]
        outs = []
        for (_, graph, flow), x in zip(loops, (x1, x2)):
            if x.requires_grad:
                flow = flow + (x.detach() - x)
            outs.append(train.flot_refine(self.refine_block, flow, graph))
        return tuple(outs)
