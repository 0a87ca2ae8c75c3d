"""Drop-in `model` package: the reference's import paths (`from model.RAFTSceneFlow import RSF`, tools/engine.py:17,
test.py:14) resolve to the H100-native implementation when this repository precedes the reference on sys.path.
Evaluation (`test.py`, `torch.no_grad()`) runs the fused inference kernels; training (`train.py` -> tools/engine.py:131-147,
tools/engine_refine.py) runs the layer-by-layer path of pvraft_b200/train.py, whose forward and backward are library kernels.
Inputs must be CUDA tensors: there is no CPU fallback on either path."""
