from . import functional  # noqa: F401
from .conv import *  # noqa: F401,F403
from .pool import *  # noqa: F401,F403
from .gmt_pool import *  # noqa: F401,F403
from .skipgram import *  # noqa: F401,F403
