"""Jumanji env registration (task ids, aliases and episode limits as in
envpool/jumanji/registration.py; Game2048 and Minesweeper are the accelerated Jumanji tasks)."""
from ..registration import register

register(task_id="Game2048-v1", import_path="envpool_b200.jumanji", spec_cls="Game2048EnvSpec",
         dm_cls="Game2048DMEnvPool", gymnasium_cls="Game2048GymnasiumEnvPool",
         aliases=["Jumanji/Game2048-v1"], max_episode_steps=1000)
register(task_id="Minesweeper-v0", import_path="envpool_b200.jumanji",
         spec_cls="MinesweeperEnvSpec", dm_cls="MinesweeperDMEnvPool",
         gymnasium_cls="MinesweeperGymnasiumEnvPool", aliases=["Jumanji/Minesweeper-v0"],
         max_episode_steps=90)
