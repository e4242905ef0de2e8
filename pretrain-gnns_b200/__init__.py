"""H100-native message-passing stack for snap-stanford/pretrain-gnns (chem/model.py, bio/model.py).

Host side: drop-in `GNN` / `GINConv` / `GNN_graphpred` modules (`.chem.model`, `.bio.model`) that keep
the reference's constructor and `forward` signatures and `state_dict` keys, dispatching through a
C-ABI shared library (`csrc/` -> `libpgnn_b200.so`, declared in `include/pgnn_b200.h`) to hand-written
sm_90a CUDA kernels.  There is no CPU fallback: a forward on a host tensor raises.
"""
__all__ = ["synthetic"]
