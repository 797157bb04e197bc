"""PGX env registration (task ids, `task` and max_num_players as in envpool/pgx/registration.py;
TicTacToe, ConnectFour, Hex, Othello, Go, Chess and GardnerChess are the accelerated PGX games;
ChineseGo*-v1 is not registered: its rules are not accelerated)."""
from ..registration import register

register(task_id="TicTacToe-v1", import_path="envpool_b200.pgx", spec_cls="TicTacToeEnvSpec",
         dm_cls="TicTacToeDMEnvPool", gymnasium_cls="TicTacToeGymnasiumEnvPool",
         task="tic_tac_toe", max_num_players=2)
register(task_id="ConnectFour-v1", import_path="envpool_b200.pgx",
         spec_cls="ConnectFourEnvSpec", dm_cls="ConnectFourDMEnvPool",
         gymnasium_cls="ConnectFourGymnasiumEnvPool", task="connect_four", max_num_players=2)
register(task_id="Hex-v1", import_path="envpool_b200.pgx", spec_cls="HexEnvSpec",
         dm_cls="HexDMEnvPool", gymnasium_cls="HexGymnasiumEnvPool", task="hex",
         max_num_players=2)
register(task_id="Othello-v1", import_path="envpool_b200.pgx", spec_cls="OthelloEnvSpec",
         dm_cls="OthelloDMEnvPool", gymnasium_cls="OthelloGymnasiumEnvPool", task="othello",
         max_num_players=2)
for _size in (9, 13, 19):
    register(task_id=f"Go{_size}x{_size}-v1", import_path="envpool_b200.pgx",
             spec_cls="GoEnvSpec", dm_cls="GoDMEnvPool", gymnasium_cls="GoGymnasiumEnvPool",
             board_size=_size, komi=7.5, history_length=8, max_terminal_steps=0, rules="pgx",
             task=f"go_{_size}x{_size}", max_num_players=2)
register(task_id="Chess-v1", import_path="envpool_b200.pgx", spec_cls="ChessEnvSpec",
         dm_cls="ChessDMEnvPool", gymnasium_cls="ChessGymnasiumEnvPool", task="chess",
         max_num_players=2)
register(task_id="GardnerChess-v1", import_path="envpool_b200.pgx", spec_cls="GardnerChessEnvSpec",
         dm_cls="GardnerChessDMEnvPool", gymnasium_cls="GardnerChessGymnasiumEnvPool",
         task="gardner_chess", max_num_players=2)
