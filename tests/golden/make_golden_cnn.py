#!/usr/bin/env python
"""Generate the convolutional-evaluate golden fixtures from the UNMODIFIED reference.

Same protocol as make_golden_seq.py (the shims and the ``run_reference`` driver of make_golden.py): the agent is
``estorch_b200.DeviceAgent``, whose ``rollout(policy)`` runs the policy on the image batch with plain torch; the
policies are ``_cnn_oracle.policy_class``: an ``nn.Sequential`` of Conv2d / activation / Flatten / Linear layers
built from the packed ``dims`` of ``CNNSpec``.  To the reference they are just another policy and agent.  Writes
only:

    es_cnn_p16.npz      classic ES, 1x12x12 images, conv 4 k3 s2 p1 / conv 6 k3 s2 / Linear 8 / Linear 4, ReLU
                        hidden, Tanh output, squared error against targets in (-0.5, 0.5), B = 6, P = 16,
                        sigma 0.05, 3 generations
    nsr_cnn_xent_p8.npz NSR-ES, 1x12x12 images, conv 3 k5 s1 p2 / conv 4 k3 s2 p1 / Linear 4, Tanh hidden,
                        identity output, cross-entropy on the blob-quadrant task, B = 8, P = 8, sigma 0.02,
                        4 generations, 8-D BC (the logits of the first 2 images)

    python tests/golden/make_golden_cnn.py
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as mg  # noqa: E402  (installs the reference shims on import)
from _cnn_oracle import image_task, pack, param_count, policy_class  # noqa: E402
from estorch_b200 import DeviceAgent  # noqa: E402

SHAPE = (1, 12, 12)
ES_DIMS = pack(SHAPE, [(4, 3, 2, 1), (6, 3, 2, 0)], [8, 4])
NSR_DIMS = pack(SHAPE, [(3, 5, 1, 2), (4, 3, 2, 1)], [4])


class DeviceXent(DeviceAgent):
    """run_reference hands its agent obs / target / bc_obs / bc_dim only: the cross-entropy form."""
    def __init__(self, obs, target, bc_obs=0, bc_dim=0):
        super().__init__(obs, target, bc_obs, bc_dim, loss="cross_entropy")


def es_data():
    obs, tgt = image_task(6, SHAPE, seed=91)
    return obs, tgt - 0.5


def nsr_data():
    return image_task(8, SHAPE, seed=92)


def run(n_conv, hidden, out_tanh, cls, agent, dims, P, sigma, n_gen, table, noise_seed, obs, target, **kw):
    mg.MLP = policy_class(n_conv, hidden, out_tanh)
    mg.SynthAgent = agent
    # run_reference sizes each noise row with orc.mlp_param_count(dims): give it the CNN's count
    orc = mg.orc
    mg.orc = types.SimpleNamespace(mlp_param_count=lambda d: param_count(d, n_conv), noise_offsets=orc.noise_offsets)
    try:
        return mg.run_reference(cls, list(dims), P, sigma, n_gen, table, noise_seed, obs, target, **kw)
    finally:
        mg.orc = orc


def main():
    obs, target = es_data()
    out = run(2, "relu", True, mg.ref.ES, DeviceAgent, ES_DIMS, 16, 0.05, 3, mg.make_table(1 << 14, 91), 71,
              obs, target)
    np.savez_compressed(os.path.join(HERE, "es_cnn_p16.npz"), **out)
    obs, target = nsr_data()
    out = run(2, "tanh", False, mg.ref.NSR_ES, DeviceXent, NSR_DIMS, 8, 0.02, 4, mg.make_table(1 << 14, 92), 73,
              obs, target, bc_obs=2, bc_dim=8)
    np.savez_compressed(os.path.join(HERE, "nsr_cnn_xent_p8.npz"), **out)
    for f in ("es_cnn_p16.npz", "nsr_cnn_xent_p8.npz"):
        print(f"  {f}: {os.path.getsize(os.path.join(HERE, f)) / 1024:.1f} KB")


if __name__ == "__main__":
    main()
