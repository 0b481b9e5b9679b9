from .config import *  # noqa: F401,F403
