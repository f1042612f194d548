from .graph_op import *  # noqa: F401,F403
from .skipgram import *  # noqa: F401,F403
