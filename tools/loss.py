"""Drop-in for the reference's tools/loss.py (same names and signatures) on the device-side kernels: with this repository
ahead of the reference on PYTHONPATH, `from tools.loss import sequence_loss` (tools/engine.py:19) resolves here.  The
self-supervised losses take the same arguments and read only batch['sequence'], so an engine trains without ground truth by
importing sequence_self_supervised_loss (or self_supervised_loss) under the name it uses.  Both also take the (forward,
backward) pair of a bidirectional forward, with the forward-backward consistency term's w_consistency and k_cons."""
from pvraft_b200.loss import (compute_loss, self_supervised_loss, sequence_loss,  # noqa: F401
                              sequence_self_supervised_loss)
