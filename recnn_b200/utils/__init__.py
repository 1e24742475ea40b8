from . import metrics, misc
from .diversify import diversify
from .misc import soft_update, write_losses, DummyWriter
