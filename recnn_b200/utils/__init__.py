from . import metrics, misc
from .misc import soft_update, write_losses, DummyWriter
