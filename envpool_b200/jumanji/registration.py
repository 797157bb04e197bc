"""Jumanji env registration (task id, alias and episode limit as in
envpool/jumanji/registration.py; Game2048 is the one accelerated Jumanji task)."""
from ..registration import register

register(task_id="Game2048-v1", import_path="envpool_b200.jumanji", spec_cls="Game2048EnvSpec",
         dm_cls="Game2048DMEnvPool", gymnasium_cls="Game2048GymnasiumEnvPool",
         aliases=["Jumanji/Game2048-v1"], max_episode_steps=1000)
