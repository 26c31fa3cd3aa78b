"""The part of the reference's gluon package that sits between Trainer.allreduce_grads() and
Trainer.update(): gluon.utils.clip_global_norm."""
from . import utils
