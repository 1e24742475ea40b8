from . import models, update, algo, beta
from .models import Actor, Critic, DiscreteActor
from .algo import Algo, DDPG, TD3, Reinforce
from .beta import Beta
from .update import (temporal_difference, value_update, ddpg_update, td3_update, reinforce_update,
                     ChooseREINFORCE)
