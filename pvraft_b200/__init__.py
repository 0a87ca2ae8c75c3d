"""pvraft_b200 -- H100-native (sm_90a) implementation of PV-RAFT's per-iteration hot path behind the
reference's own nn.Module API.  See DESIGN.md; the C ABI is include/pvraft_b200.h."""
from .corr import CorrBlock
from .extractor import FlotEncoder
from .gconv import SetConv
from .graph import Graph
from .loss import flow_consistency
from .pointconv import knn_point, square_distance
from .raft import RSF, RSF_refine
from .refine import FlotRefine
from .rigid import RigidMotion, rigid_motion
from .stream import SceneFlowStream
from .update import ConvGRU, ConvRNN, FlowHead, MotionEncoder, UpdateBlock

__all__ = ['RSF', 'RSF_refine', 'CorrBlock', 'UpdateBlock', 'MotionEncoder', 'ConvGRU', 'ConvRNN', 'FlowHead',
           'FlotEncoder', 'FlotRefine', 'SetConv', 'Graph', 'knn_point', 'square_distance', 'SceneFlowStream',
           'flow_consistency', 'rigid_motion', 'RigidMotion']
