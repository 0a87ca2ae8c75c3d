"""Scene flow along a scan sequence.

`SceneFlowStream(model, num_iters)` takes the scans of a sequence one at a time and returns, for every scan after the first,
what `model([previous scan, scan], num_iters, flow_init=...)` returns.  It saves two things that separate pair calls repeat:

* every scan is encoded once.  `RSF._encode_cloud` (the feature encoder and the kNN graph with its Morton order) does not
  depend on which side of a pair a cloud is on: a scan's feature map is `fmap2` of the pair that ends with it, and its
  feature map and graph are `fmap1` and pc1's graph of the next pair.  The correlation build, the context encoder and the
  loop (`RSF._pair`, `RSF._run`) run per pair as in `forward`.
* with `warm_start`, the loop starts from the motion already estimated: from the third scan on, the previous pair's final
  flow (on its first cloud) is carried onto the current first cloud by `ops.flow_propagate` and passed as `flow_init`.

CUDA graphs follow the model's policy (`use_cuda_graph`, PVRAFT_CUDA_GRAPH): batches of at most 2 samples replay from the
first step, larger batches from the second step with the same shapes and weights.  One step is one replay, the propagation
included: the cached scan state is copied into the graph's static buffers and the new scan's state copied back out.
"""
import torch

from . import ops
from ._lib import PvraftError
from .graph import Graph

_MAX_GRAPHS = 8


def _scan_state(fmap, graph):
    """What a stream keeps of an encoded scan besides its points: the feature map and the kNN graph's tensors."""
    state = {'fmap': fmap, 'nbr': graph.nbr, 'rel': graph._rel, 'plan': graph.plan}
    if graph.order is not None:
        state['order'] = graph.order
    return state


class SceneFlowStream:
    """Inference along a scan sequence with `model` (an `RSF` or `RSF_refine`), `num_iters` RAFT iterations per pair.

    step(xyz [B,N_t,3]) -> None for the first scan; then the model's output for the pair (previous scan, xyz): the list of
    num_iters flows [B,N_{t-1},3] for RSF, the refined flow for RSF_refine.  Scan sizes may change from step to step; every
    pair obeys ops.check_pair.  warm_start: from the third scan on, the pair starts at flow_init = ops.flow_propagate(first
    cloud of the previous pair, its final flow, first cloud of this pair, k); the second scan starts cold.  reset() forgets
    the sequence.  Steps run under torch.no_grad() (the stream does not train)."""

    def __init__(self, model, num_iters, warm_start=True, k=3):
        if isinstance(model, torch.nn.DataParallel):
            raise TypeError('SceneFlowStream runs one module: pass model.module, not the nn.DataParallel wrapper')
        if not all(hasattr(model, a) for a in ('_encode_cloud', '_pair', '_run')):
            raise TypeError(f'SceneFlowStream needs an RSF or RSF_refine, got {type(model).__name__}')
        if isinstance(k, bool) or not isinstance(k, int) or not 1 <= k <= ops.PROPAGATE_MAX_K:
            raise ValueError(f'k={k!r} must be an integer in 1..{ops.PROPAGATE_MAX_K}')
        if isinstance(num_iters, bool) or not isinstance(num_iters, int) or num_iters < 1:
            raise ValueError(f'num_iters={num_iters!r} must be a positive integer')
        self.model, self.num_iters, self.warm_start, self.k = model, num_iters, bool(warm_start), k
        self.reset()

    def reset(self):
        self._scan = None   # the last scan: {'xyz', 'fmap', 'nbr', 'rel', 'plan'[, 'order']}
        self._stamp = None  # the model's parameters when that scan was encoded
        self._last = None   # the last pair: (its first cloud, its final flow on that cloud)

    def step(self, xyz):
        if not torch.is_tensor(xyz) or xyz.dim() != 3 or xyz.shape[-1] != 3:
            raise ValueError(f'expected a scan [B,N,3], got {tuple(xyz.shape) if torch.is_tensor(xyz) else type(xyz).__name__}')
        if self._scan is None:
            ops.check_pair(xyz, xyz, 0)
        else:
            ops.check_pair(self._scan['xyz'], xyz, self.model.corr_block.truncate_k)
        if not xyz.is_cuda:
            raise PvraftError('pvraft_b200 kernels need CUDA tensors (no CPU fallback exists)')
        if self._scan is not None and xyz.device != self._scan['xyz'].device:
            raise PvraftError(f'scan on {xyz.device}, the sequence on {self._scan["xyz"].device}')
        m = self.model
        with torch.no_grad(), torch.cuda.device(xyz.device):
            stamp = m._stamp()
            if self._scan is not None and self._stamp != stamp:
                # the weights changed since the last scan was encoded (load_state_dict, an optimizer step): encode it again
                self._scan = dict(xyz=self._scan['xyz'], **_scan_state(*m._encode_cloud(self._scan['xyz'])))
            state = {'xyz': xyz.detach().float().contiguous().clone()}   # (kept as the next pair's first cloud)
            if self._scan is not None:
                state.update({k + '1': v for k, v in self._scan.items()})
                if self.warm_start and self._last is not None:
                    state['src_xyz'], state['src_flow'] = self._last
            if self._use_graph(state, stamp):
                out, new = self._replay(state, stamp)
            else:
                out, new = self._body(state)
            if out is not None:
                final = out[-1] if isinstance(out, (list, tuple)) else out
                self._last = (self._scan['xyz'], final.clone())
            self._scan, self._stamp = dict(xyz=state['xyz'], **new), stamp
        return out

    # -- one step: the work a replay records ------------------------------------------------------------------------------------
    def _body(self, s):
        """s: the new scan 'xyz', the previous scan's state (keys ending in 1) and, warm, 'src_xyz' / 'src_flow' -> (the
        model's output or None, the new scan's state)."""
        m = self.model
        fmap, graph = m._encode_cloud(s['xyz'])
        new = _scan_state(fmap, graph)
        if 'xyz1' not in s:
            return None, new
        xyz1 = s['xyz1']
        b, n1, _ = xyz1.shape
        graph1 = Graph(s['nbr1'], s['rel1'], ops.KNN, [b * n1] * 2, s.get('order1'), s['plan1'])
        flow_init = ops.flow_propagate(s['src_xyz'], s['src_flow'], xyz1, self.k) if 'src_xyz' in s else None
        return m._run(m._pair(xyz1, s['xyz'], s['fmap1'], graph1, fmap), self.num_iters, flow_init), new

    # -- CUDA graphs -------------------------------------------------------------------------------------------------------------
    def _key(self, s):
        m = self.model
        shapes = tuple((k, tuple(s[k].shape)) for k in ('xyz1', 'xyz', 'src_xyz') if k in s)
        precision = (m.corr_block.state_dtype, bool(m.bf16_compute))
        return (shapes, s['xyz'].device, self.num_iters, ops.deterministic(), 'src_xyz' in s, self.k if 'src_xyz' in s else 0,
                precision)

    def _use_graph(self, s, stamp):
        m = self.model
        graph = m.use_cuda_graph
        if graph is not None:
            return bool(graph)
        if s['xyz'].shape[0] <= 2:
            return True                            # host-bound from the first step
        seen = m.__dict__.setdefault('_stream_seen', {})
        key = self._key(s)
        again = seen.get(key) == stamp             # the same shapes came back with the same weights
        if len(seen) > 64:
            seen.clear()
        seen[key] = stamp
        return again

    def _replay(self, s, stamp):
        """The step as one replay of a graph kept on the model (invalidated with its own graphs: a weight change or
        set_precision), at most _MAX_GRAPHS of them."""
        m = self.model
        graphs = m.__dict__.setdefault('_stream_graphs', {})
        key = self._key(s)
        entry = graphs.get(key)
        if entry is not None and entry[3] != stamp:
            entry = None                           # weights changed since the capture: stale derived constants
        if entry is None:
            static = {k: v.clone() for k, v in s.items()}
            dev = s['xyz'].device
            side = torch.cuda.Stream(device=dev)   # warm-up off the capture stream: weight splits, derived constants
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):
                for _ in range(2):
                    self._body(static)
            torch.cuda.current_stream(dev).wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            l0 = ops.launch_count
            with torch.cuda.graph(graph):
                static_out = self._body(static)
            graphs.pop(key, None)
            while len(graphs) >= _MAX_GRAPHS:      # oldest capture out (its private memory pool goes with it)
                graphs.pop(next(iter(graphs)))
            entry = graphs[key] = (graph, static, static_out, stamp, ops.launch_count - l0)
        graph, static, (out, new), _, n_kernels = entry
        for k, v in s.items():
            static[k].copy_(v)
        graph.replay()
        ops.launch_count += n_kernels              # the library's kernels inside the replayed graph
        if out is not None:
            out = out.clone() if torch.is_tensor(out) else [t.clone() for t in out]
        return out, {k: v.clone() for k, v in new.items()}
