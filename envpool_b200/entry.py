"""Entry point for all envs' registration (mirror of envpool/entry.py)."""
from .classic_control import registration as _cc  # noqa: F401
from .jumanji import registration as _jm  # noqa: F401
from .mujoco.gym import registration as _mg  # noqa: F401
from .pgx import registration as _pgx  # noqa: F401
from .toy_text import registration as _tt  # noqa: F401
