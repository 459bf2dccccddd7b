"""TEST-ONLY: population mode of a generic convolutional policy (estk_act_cnn, include/estk_act_cnn.h): the small
pixel agent of the CPU tests and the goldens, and the goldens' policy shapes."""
import torch

from _cnn_oracle import pack, param_count, policy_class
from estorch_b200 import PopulationAgent

ACTIONS = 3 << 16        # include/estk.h ESTK_ACTIONS
OBS_SHAPE = (2, 8, 8)
# the goldens' policies: conv 2->4 k3 pad 1, conv 4->8 k3 s2, flatten (8x3x3), Linear 72->16, Linear 16->2
DIMS = pack(OBS_SHAPE, [(4, 3, 1, 1), (8, 3, 2, 0)], [16, 2])
N_PARAMS = param_count(DIMS, 2)
ES_POLICY = dict(n_conv=2, hidden="relu", out_tanh=True)      # es_pop_cnn_p16.npz
NSR_POLICY = dict(n_conv=2, hidden="elu", out_tanh=False)     # nsr_pop_cnn_p8.npz


def cnn_policy(n_conv, hidden, out_tanh):
    """The policy class (``__init__(dims)``, an ``nn.Sequential`` with ``nn.Flatten``) of a golden."""
    return policy_class(n_conv, hidden, out_tanh)


class PixelPoint(PopulationAgent):
    """A point in the plane rendered into 2x8x8 images: channel 0 a Gaussian blob at the point, channel 1 one at
    the goal.  The two outputs move it smoothly, s' = s + 0.1 * tanh(y), no argmax, so fp32 order differences
    in the forward stay in the last bits of the returns; reward -|s' - goal|^2 per step, fixed start and
    horizon.  Vectorised over members; one image per member and step, so the reference protocol
    ``rollout(policy)`` hands a plain Conv2d stack ``[1, 2, 8, 8]``.  ``bc_dim`` = 4 makes it an NS-family
    agent: the point at the middle and at the end."""

    obs_shape = OBS_SHAPE

    def __init__(self, horizon=6, bc_dim=0):
        assert bc_dim in (0, 4)
        self.horizon, self.bc_dim = horizon, bc_dim
        self.s0 = torch.tensor([-0.5, 0.4])
        self.goal = torch.tensor([0.3, -0.2])

    def frames(self, s):
        """[M, 2] points -> [M, 2, 8, 8] float32 images."""
        g = (torch.arange(8, device=s.device, dtype=torch.float32) + 0.5) / 4.0 - 1.0
        goal = self.goal.to(s.device).expand_as(s)
        blobs = []
        for p in (s, goal):
            d2 = (g[None, :, None] - p[:, 0, None, None]) ** 2 + (g[None, None, :] - p[:, 1, None, None]) ** 2
            blobs.append(torch.exp(-d2 / (2 * 0.3 ** 2)))
        return torch.stack(blobs, 1).contiguous()

    def rollout_population(self, act, members):
        dev = self.device
        s = self.s0.to(dev).expand(members, 2).contiguous()
        goal = self.goal.to(dev)
        ret = torch.zeros(members, device=dev)
        mid = s
        for t in range(self.horizon):
            y = act(self.frames(s))
            s = s + 0.1 * torch.tanh(y)
            ret = ret - ((s - goal) ** 2).sum(1)
            if t + 1 == self.horizon // 2:
                mid = s
        if self.bc_dim:
            return ret, torch.cat([mid, s], 1)
        return ret
