"""Drop-in for the reference's src/discriminators.py: PoseDiscriminator over human_dynamics_b200.adversarial (CUDA)."""
from human_dynamics_b200 import adversarial


class PoseDiscriminator(object):
    def __init__(self, weight_decay, weights=None, seed=0):
        """weight_decay is kept for the reference's signature; like the reference's trainer, nothing applies it.  weights / seed: the
        variables' values (adversarial.PoseDiscriminator), used when the first get_output creates them."""
        self.vars = []
        self.reuse = False
        self.wd = weight_decay
        self.net = None
        self._init = (weights, seed)

    def get_output(self, poses):
        """poses (N, 23, 1, 9) or (N, 23, 9) CUDA float32 -> predictions (N, 24): one per joint, then one for the whole pose."""
        if not self.reuse:
            self.net = adversarial.PoseDiscriminator(self._init[0], seed=self._init[1], device=poses.device)
            self.update(list(self.net.parameters()))
        return self.net(poses)

    def get_vars(self):
        return self.vars

    def update(self, vars):
        self.reuse = True
        self.vars.extend(vars)
