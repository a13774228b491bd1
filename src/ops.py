"""src/ops.py of the reference holds the training losses and a duplicate of the IEF wrappers (ops.py:184,270).  BASELINE.json names
`src/ops.batch_orth_proj_idrot`; export it here as an alias.  The adversarial prior's losses (ops.py:127-137, 160) are torch expressions
over the discriminator's outputs (src/discriminators.py) and the predicted shapes."""
from src.tf_smpl.projection import batch_orth_proj_idrot  # noqa: F401
from src.models import call_hmr_ief, hmr_ief              # noqa: F401


def compute_loss_e_fake(out_fake):
    return ((out_fake - 1) ** 2).sum(dim=1).mean()


def compute_loss_d_fake(out_fake):
    return (out_fake ** 2).sum(dim=1).mean()


def compute_loss_d_real(out_real):
    return ((out_real - 1) ** 2).sum(dim=1).mean()


def compute_loss_shape(shapes):
    """L2 loss on shapes."""
    return shapes.square().mean()
