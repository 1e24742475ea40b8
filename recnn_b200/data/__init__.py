from . import utils, env, feed, db_con, item_sets
from .utils import (rolling_window, batch_tensor_embeddings, batch_contstate_discaction, batch_frames,
                    prepare_batch_static_size,
                    make_items_tensor, get_base_batch)
from .env import UserDataset, EnvBase, DataPath, Env, FrameEnv
from .feed import HistoryCSR, DeviceFrameFeed
from .db_con import ItemIndex, SearchResult, MilvusConnection
from .item_sets import ItemSets
