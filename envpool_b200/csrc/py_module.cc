// pybind11 host modules: the drop-in replacement for the class pairs the reference
// generates with REGISTER(m, SPEC, ENVPOOL) (envpool/core/py_envpool.h:303-332) in
// classic_control/classic_control.cc, toy_text/toy_text.cc, jumanji/jumanji_envpool.cc,
// mujoco/gym/mujoco_envpool.cc and pgx/pgx.cc.
// Same class names (_XxxEnvSpec / _XxxEnvPool), same attributes, same tuple formats, so the
// reference's own Python layer (envpool/python/api.py:22-41 py_env()) can sit on top of it
// unchanged.  Everything below the boundary is the C ABI of include/envpool_b200.h --
// no env arithmetic lives in this file.
//
// Built five times (one module per reference family) with -DEPB_FAMILY_* selecting the
// env list; see envpool_b200/_build.py.
#include <pybind11/numpy.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdlib>
#include <cstdint>
#include <memory>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

#include "envpool_b200.h"

namespace py = pybind11;

namespace {

struct Col {
  std::string key;
  char dtype;  // 'i' int32, 'f' float32, 'd' float64, 'b' bool
  std::vector<int> shape;
  bool has_bounds = false;
  double lo = 0, hi = 0;
  std::vector<double> lo_vec, hi_vec;
};

py::dtype np_dtype(char c) {
  switch (c) {
    case 'i': return py::dtype::of<int>();
    case 'f': return py::dtype::of<float>();
    case 'd': return py::dtype::of<double>();
    default: return py::dtype::of<bool>();
  }
}

// (dtype, shape, (lo, hi), (lo_vec, hi_vec), is_discrete): SpecTupleHelper::Make,
// py_envpool.h:103-110.  Unbounded specs carry numeric_limits<T>::min()/max() exactly as
// core/spec.h:67-68 does (so float "min" is FLT_MIN, the reference's quirk).
py::tuple export_col(const Col& c) {
  py::object lo, hi, lov, hiv;
  auto vec = [&](const std::vector<double>& v) -> py::object {
    py::list l;
    for (double x : v) {
      if (c.dtype == 'i') l.append(py::int_(static_cast<int>(x)));
      else if (c.dtype == 'f') l.append(py::float_(static_cast<double>(static_cast<float>(x))));
      else l.append(py::float_(x));
    }
    return std::move(l);
  };
  switch (c.dtype) {
    case 'i':
      lo = py::int_(c.has_bounds ? static_cast<int>(c.lo) : INT_MIN);
      hi = py::int_(c.has_bounds ? static_cast<int>(c.hi) : INT_MAX);
      break;
    case 'f':
      lo = py::float_(c.has_bounds ? static_cast<double>(static_cast<float>(c.lo)) : static_cast<double>(FLT_MIN));
      hi = py::float_(c.has_bounds ? static_cast<double>(static_cast<float>(c.hi)) : static_cast<double>(FLT_MAX));
      break;
    case 'd':
      lo = py::float_(c.has_bounds ? c.lo : DBL_MIN);
      hi = py::float_(c.has_bounds ? c.hi : DBL_MAX);
      break;
    default:
      lo = py::bool_(false);
      hi = py::bool_(true);
  }
  return py::make_tuple(np_dtype(c.dtype), c.shape, py::make_tuple(lo, hi),
                        py::make_tuple(vec(c.lo_vec), vec(c.hi_vec)), false);
}

Col col(const std::string& k, char d, std::vector<int> shape) {
  Col c;
  c.key = k;
  c.dtype = d;
  c.shape = std::move(shape);
  return c;
}
Col colb(const std::string& k, char d, std::vector<int> shape, double lo, double hi) {
  Col c = col(k, d, std::move(shape));
  c.has_bounds = true;
  c.lo = lo;
  c.hi = hi;
  return c;
}
Col colv(const std::string& k, char d, std::vector<int> shape, std::vector<double> lo,
         std::vector<double> hi) {
  Col c = col(k, d, std::move(shape));
  c.lo_vec = std::move(lo);
  c.hi_vec = std::move(hi);
  return c;
}

// Static description of one env class: config keys/defaults and the spec builders.
struct EnvDesc {
  const char* name;  // reference class stem, e.g. "CartPole"
  int kind;
  std::vector<std::string> cfg_keys;   // env-specific keys (XxxEnvFns::DefaultConfig)
  py::tuple (*cfg_defaults)();
  int players = 1;  // players per env: the max_num_players a pool of this kind must be given
};

constexpr int kNumCommon = 10;
const char* kCommonKeys[kNumCommon] = {
    // common_config, envpool/core/env_spec.h:26-31
    "num_envs", "batch_size", "num_threads", "max_num_players", "thread_affinity_offset",
    "base_path", "seed", "env_seed", "gym_reset_return_info", "max_episode_steps"};
py::tuple common_defaults() {
  return py::make_tuple(1, 0, 0, 1, -1, std::string("envpool"), 42, std::vector<int>{}, true,
                        INT_MAX);
}

// Game2048's board strings (jumanji/game2048_env.h ParseBoard, parse::CsvArray): comma-separated
// integers, the first `n` of them used, missing cells 0; a token that is not a number raises
// ValueError, as std::stoi / std::stoll do.  Empty text = not configured (an empty vector).
std::vector<int32_t> parse_cells(const std::string& text, int n, const char* key) {
  std::vector<int32_t> cells;
  if (text.empty()) return cells;
  cells.assign(n, 0);
  std::stringstream stream(text);
  std::string token;
  int index = 0;
  while (index < n && std::getline(stream, token, ',')) {
    try {
      cells[index++] = static_cast<int32_t>(std::stoll(token));
    } catch (const std::exception&) {
      throw std::invalid_argument(std::string(key) + ": '" + token + "' is not an integer");
    }
  }
  for (int32_t v : cells)
    if (v < 0 || v > 26)
      throw std::invalid_argument(std::string(key) + ": cell " + std::to_string(v) +
                                  " is not a tile exponent in [0, 26]");
  return cells;
}

// Minesweeper's config strings, read with the reference's own calls and token rules
// (jumanji/minesweeper_env.h ParseMineLocations, jumanji/parse_utils.h CsvArray), so every string
// the reference accepts reads identically; where std::stoi / std::stoll / std::stof throw, the
// reference throws too, and so does this (ValueError).
struct MinesweeperConfig {
  std::vector<int32_t> mines;    // 100 cells, 1 = mine; empty = random placement
  std::vector<int32_t> boards;   // 32 x 100 cells, missing ones -1
  std::vector<float> rewards;    // 32, missing ones 0.0f
  std::vector<uint8_t> done;     // 32, missing ones false
  bool replay = false;           // minesweeper_replay_boards is not empty
};
template <typename T, typename Read>
std::vector<T> csv_array(const std::string& text, size_t n, T fill, const char* key, Read read) {
  std::vector<T> values(n, fill);
  if (text.empty()) return values;
  std::stringstream stream(text);
  std::string token;
  size_t index = 0;
  while (std::getline(stream, token, ',') && index < n) {
    try {
      values[index++] = read(token);
    } catch (const std::exception&) {
      throw std::invalid_argument(std::string(key) + ": cannot read '" + token + "'");
    }
  }
  return values;
}
MinesweeperConfig parse_minesweeper(const std::string& mines, const std::string& boards,
                                    const std::string& rewards, const std::string& done) {
  MinesweeperConfig c;
  if (!mines.empty()) {
    c.mines.assign(100, 0);
    bool any = false;
    std::stringstream stream(mines);
    std::string token;
    while (std::getline(stream, token, ',')) {
      int location;
      try {
        location = std::stoi(token);
      } catch (const std::exception&) {
        throw std::invalid_argument("minesweeper_mine_locations: cannot read '" + token + "'");
      }
      if (0 <= location && location < 100) {  // others are dropped, duplicates merge
        c.mines[location] = 1;
        any = true;
      }
    }
    if (!any) c.mines.clear();  // nothing in range: random placement, as for an empty string
  }
  c.boards = csv_array<int32_t>(boards, 32 * 100, -1, "minesweeper_replay_boards",
                                [](const std::string& t) { return static_cast<int32_t>(std::stoll(t)); });
  for (int32_t v : c.boards)
    if (v < -1 || v > 8)
      throw std::invalid_argument("minesweeper_replay_boards: cell " + std::to_string(v) +
                                  " is not a Minesweeper cell in [-1, 8]");
  c.rewards = csv_array<float>(rewards, 32, 0.0f, "minesweeper_replay_rewards",
                               [](const std::string& t) { return std::stof(t); });
  c.done = csv_array<uint8_t>(done, 32, 0, "minesweeper_replay_done", [](const std::string& t) {
    return static_cast<uint8_t>(t == "1" || t == "True" || t == "true");
  });
  c.replay = !boards.empty();
  return c;
}

class SpecBase {
 public:
  const EnvDesc* desc;
  py::tuple config_values;
  std::vector<Col> state_cols, action_cols;
  std::vector<int32_t> game2048_initial, game2048_replay;  // parsed board strings
  MinesweeperConfig minesweeper;

  SpecBase(const EnvDesc* d, const py::tuple& conf) : desc(d) {
    const size_t want = kNumCommon + d->cfg_keys.size();
    if (conf.size() != want)
      throw std::invalid_argument("config tuple has " + std::to_string(conf.size()) +
                                  " values, expected " + std::to_string(want));
    int num_envs = conf[0].cast<int>(), batch = conf[1].cast<int>();
    // EnvSpec ctor, envpool/core/env_spec.h:75-83
    if (batch > num_envs)
      throw std::invalid_argument(
          "It is required that batch_size <= num_envs, got num_envs = " +
          std::to_string(num_envs) + ", batch_size = " + std::to_string(batch));
    py::list l;
    for (size_t i = 0; i < conf.size(); ++i) l.append(conf[i]);
    if (batch == 0) l[1] = py::int_(num_envs);
    config_values = py::tuple(l);
    // common_state_spec / common_action_spec, env_spec.h:34-43
    state_cols = {col("info:env_id", 'i', {}), col("info:players.env_id", 'i', {-1}),
                  col("elapsed_step", 'i', {}), col("done", 'b', {}),
                  col("reward", 'f', {-1}), colb("discount", 'f', {-1}, 0.0, 1.0),
                  col("step_type", 'i', {}), col("trunc", 'b', {})};
    action_cols = {col("env_id", 'i', {}), col("players.env_id", 'i', {-1})};
    BuildEnvCols();
  }
  template <typename T>
  T cfg(const std::string& key) const {
    for (int i = 0; i < kNumCommon; ++i)
      if (key == kCommonKeys[i]) return config_values[i].cast<T>();
    for (size_t i = 0; i < desc->cfg_keys.size(); ++i)
      if (key == desc->cfg_keys[i]) return config_values[kNumCommon + i].cast<T>();
    throw std::out_of_range("no config key " + key);
  }
  py::tuple StateSpecPy() const {
    py::list l;
    for (auto& c : state_cols) l.append(export_col(c));
    return py::tuple(l);
  }
  py::tuple ActionSpecPy() const {
    py::list l;
    for (auto& c : action_cols) l.append(export_col(c));
    return py::tuple(l);
  }
  std::vector<std::string> StateKeys() const {
    std::vector<std::string> k;
    for (auto& c : state_cols) k.push_back(c.key);
    return k;
  }
  std::vector<std::string> ActionKeys() const {
    std::vector<std::string> k;
    for (auto& c : action_cols) k.push_back(c.key);
    return k;
  }

 private:
  void BuildEnvCols() {
    const double inf = std::numeric_limits<double>::infinity();
    const double pi = 3.14159265358979323846;
    switch (desc->kind) {
      case EPB_CARTPOLE:  // classic_control/cartpole.h:38-47
        state_cols.push_back(colv("obs", 'f', {4}, {-4.8, -inf, -pi / 7.5, -inf},
                                  {4.8, inf, pi / 7.5, inf}));
        action_cols.push_back(colb("action", 'i', {-1}, 0, 1));
        break;
      case EPB_PENDULUM:  // pendulum.h:35-44
        state_cols.push_back(colv("obs", 'f', {3}, {-1.0, -1.0, -8.0}, {1.0, 1.0, 8.0}));
        action_cols.push_back(colb("action", 'f', {-1, 1}, -2.0, 2.0));
        break;
      case EPB_ACROBOT:  // acrobot.h:37-49
        state_cols.push_back(colv("obs", 'f', {6}, {-1.0, -1.0, -1.0, -1.0, -4 * pi, -9 * pi},
                                  {1.0, 1.0, 1.0, 1.0, 4 * pi, 9 * pi}));
        state_cols.push_back(col("info:state", 'f', {2}));
        action_cols.push_back(colb("action", 'i', {-1}, 0, 2));
        break;
      case EPB_MOUNTAIN_CAR:  // mountain_car.h:37-46
        state_cols.push_back(colv("obs", 'f', {2}, {-1.2, -0.07}, {0.6, 0.07}));
        action_cols.push_back(colb("action", 'i', {-1}, 0, 2));
        break;
      case EPB_MOUNTAIN_CAR_CONTINUOUS:  // mountain_car_continuous.h:37-46
        state_cols.push_back(colv("obs", 'f', {2}, {-1.2, -0.07}, {0.6, 0.07}));
        action_cols.push_back(colb("action", 'f', {-1, 1}, -1.0, 1.0));
        break;
      case EPB_FROZEN_LAKE: {  // toy_text/frozen_lake.h:38-46
        int size = cfg<int>("size");
        state_cols.push_back(colb("obs", 'i', {-1}, 0, size * size - 1));
        action_cols.push_back(colb("action", 'i', {-1}, 0, 3));
        break;
      }
      case EPB_CATCH: {  // catch.h:36-45
        int h = cfg<int>("height"), w = cfg<int>("width");
        if (h != 10 || w != 5)
          throw std::invalid_argument(
              "Catch: only the registered height=10, width=5 board is accelerated");
        state_cols.push_back(colb("obs", 'f', {h, w}, 0.0, 1.0));
        action_cols.push_back(colb("action", 'i', {-1}, 0, 2));
        break;
      }
      case EPB_TAXI:  // taxi.h:36-43
        state_cols.push_back(colb("obs", 'i', {-1}, 0, 499));
        action_cols.push_back(colb("action", 'i', {-1}, 0, 5));
        break;
      case EPB_NCHAIN:  // nchain.h:34-41
        state_cols.push_back(colb("obs", 'i', {-1}, 0, 4));
        action_cols.push_back(colb("action", 'i', {-1}, 0, 1));
        break;
      case EPB_CLIFF_WALKING:  // cliffwalking.h:37-46
        state_cols.push_back(colb("obs", 'i', {-1}, 0, 47));
        state_cols.push_back(col("info:prob", 'f', {-1}));
        action_cols.push_back(colb("action", 'i', {-1}, 0, 3));
        break;
      case EPB_BLACKJACK:  // blackjack.h:36-43
        state_cols.push_back(colb("obs", 'i', {3}, 0, 31));
        action_cols.push_back(colb("action", 'i', {-1}, 0, 1));
        break;
      case EPB_HALF_CHEETAH: {  // mujoco/gym/half_cheetah.h:44-66
        state_cols.push_back(colb("obs", 'd', {17}, -inf, inf));
        state_cols.push_back(col("info:reward_run", 'd', {-1}));
        state_cols.push_back(col("info:reward_ctrl", 'd', {-1}));
        state_cols.push_back(col("info:x_position", 'd', {-1}));
        state_cols.push_back(col("info:x_velocity", 'd', {-1}));
        action_cols.push_back(colb("action", 'd', {-1, 6}, -1.0, 1.0));
        break;
      }
      case EPB_GAME2048:  // jumanji/game2048_env.h Game2048EnvFns
        game2048_initial = parse_cells(cfg<std::string>("game2048_initial_board"), 16,
                                       "game2048_initial_board");
        game2048_replay = parse_cells(cfg<std::string>("game2048_replay_boards"), 32 * 16,
                                      "game2048_replay_boards");
        state_cols.push_back(col("obs:board", 'i', {4, 4}));
        state_cols.push_back(colb("obs:action_mask", 'b', {4}, 0, 1));
        state_cols.push_back(colb("info:highest_tile", 'i', {}, 1, 1 << 30));
        action_cols.push_back(colb("action", 'i', {-1}, 0, 3));
        break;
      case EPB_MINESWEEPER:  // jumanji/minesweeper_env.h MinesweeperEnvFns
        minesweeper = parse_minesweeper(cfg<std::string>("minesweeper_mine_locations"),
                                        cfg<std::string>("minesweeper_replay_boards"),
                                        cfg<std::string>("minesweeper_replay_rewards"),
                                        cfg<std::string>("minesweeper_replay_done"));
        state_cols.push_back(colb("obs:board", 'i', {10, 10}, -1, 8));
        state_cols.push_back(colb("obs:action_mask", 'b', {10, 10}, 0, 1));
        state_cols.push_back(colb("obs:num_mines", 'i', {}, 0, 99));
        state_cols.push_back(colb("obs:step_count", 'i', {}, 0, 90));
        action_cols.push_back(colb("action", 'i', {-1, 2}, 0, 9));
        break;
      case EPB_TIC_TAC_TOE:  // pgx/board_games.h TicTacToeEnvFns
      case EPB_CONNECT_FOUR:  // pgx/board_games.h ConnectFourEnvFns
      case EPB_HEX:           // pgx/board_games.h HexEnvFns
      case EPB_OTHELLO: {     // pgx/board_games.h OthelloEnvFns
        const int k = desc->kind;
        const int rows = k == EPB_TIC_TAC_TOE ? 3 : k == EPB_CONNECT_FOUR ? 6 : k == EPB_HEX ? 11 : 8;
        const int cols = k == EPB_TIC_TAC_TOE ? 3 : k == EPB_CONNECT_FOUR ? 7 : rows;
        const int actions = k == EPB_TIC_TAC_TOE ? 9 : k == EPB_CONNECT_FOUR ? 7 : rows * cols + 1;
        state_cols.push_back(col("obs", 'b', {-1, rows, cols, k == EPB_HEX ? 4 : 2}));
        state_cols.push_back(col("info:board", 'i', {rows, cols}));
        state_cols.push_back(col("info:current_player", 'i', {}));
        state_cols.push_back(col("info:legal_action_mask", 'b', {actions}));
        state_cols.push_back(colb("info:players.id", 'i', {-1}, 0, 1));
        action_cols.push_back(colb("action", 'i', {-1}, 0, actions - 1));
        break;
      }
      case EPB_CHESS:           // pgx/chess_games.h ChessEnvFns
      case EPB_GARDNER_CHESS: {  // pgx/chess_games.h GardnerChessEnvFns
        const bool chess = desc->kind == EPB_CHESS;
        const int size = chess ? 8 : 5, actions = chess ? 4672 : 1225;
        state_cols.push_back(col("obs", 'f', {-1, size, size, chess ? 119 : 115}));
        state_cols.push_back(col("info:board", 'i', {size, size}));
        if (chess) state_cols.push_back(col("info:castling_rights", 'b', {2, 2}));
        state_cols.push_back(colb("info:current_player", 'i', {}, 0, 1));
        if (chess) state_cols.push_back(colb("info:en_passant", 'i', {}, -1, 63));
        state_cols.push_back(col("info:fullmove_count", 'i', {}));
        state_cols.push_back(col("info:halfmove_count", 'i', {}));
        state_cols.push_back(col("info:legal_action_mask", 'b', {actions}));
        state_cols.push_back(colb("info:players.id", 'i', {-1}, 0, 1));
        state_cols.push_back(colb("info:turn", 'i', {}, 0, 1));
        action_cols.push_back(colb("action", 'i', {-1}, 0, actions - 1));
        break;
      }
      case EPB_GO_19X19: {  // pgx/go.h GoEnvFns (every board size: go_kind picks the kernels)
        const int size = go_size(), area = size * size;
        state_cols.push_back(col("obs", 'b', {-1, size, size, 17}));
        state_cols.push_back(colb("info:board", 'i', {size, size}, -1, 1));
        state_cols.push_back(colb("info:current_player", 'i', {}, 0, 1));
        state_cols.push_back(col("info:legal_action_mask", 'b', {area + 1}));
        state_cols.push_back(colb("info:ko", 'i', {}, -1, area - 1));
        state_cols.push_back(col("info:is_psk", 'b', {}));
        state_cols.push_back(col("info:consecutive_pass_count", 'i', {}));
        state_cols.push_back(col("info:black_area", 'i', {}));
        state_cols.push_back(col("info:white_area", 'i', {}));
        state_cols.push_back(colb("info:players.id", 'i', {-1}, 0, 1));
        action_cols.push_back(colb("action", 'i', {-1}, 0, area));
        break;
      }
    }
  }

 public:
  // Go's board_size after the checks of the accelerated path (ValueError outside it): the
  // reference's boards 9, 13 and 19, history_length 8, max_terminal_steps in [0, 2 S^2] and the
  // rules "pgx" / "tromp_taylor" ("chinese" masks repeated positions, which is not accelerated)
  int go_size() const {
    const int size = cfg<int>("board_size");
    if (size != 9 && size != 13 && size != 19)
      throw std::invalid_argument("Go: board_size " + std::to_string(size) +
                                  " is not accelerated (9, 13 or 19)");
    if (cfg<int>("history_length") != 8)
      throw std::invalid_argument("Go: only history_length=8 is accelerated");
    const int steps = cfg<int>("max_terminal_steps");
    if (steps < 0 || steps > 2 * size * size)
      throw std::invalid_argument("Go: max_terminal_steps must lie in [0, 2 * board_size^2]");
    const std::string rules = cfg<std::string>("rules");
    if (rules != "pgx" && rules != "tromp_taylor")
      throw std::invalid_argument("Go: rules '" + rules +
                                  "' are not accelerated ('pgx' or 'tromp_taylor')");
    return size;
  }
  // the engine kind of the pool: Go's follows its board size
  int engine_kind() const {
    if (desc->kind != EPB_GO_19X19) return desc->kind;
    const int size = go_size();
    return size == 9 ? EPB_GO_9X9 : size == 13 ? EPB_GO_13X13 : EPB_GO_19X19;
  }
};

void check(int rc) {
  if (rc == EPB_OK) return;
  std::string msg = epb_last_error();
  if (rc == EPB_ERR_INVALID) throw std::invalid_argument(msg);
  throw std::runtime_error(msg);
}

struct PoolHandle {
  epb_pool* p = nullptr;
  ~PoolHandle() {
    if (p) epb_destroy(p);
  }
};
struct SlabLease {  // keeps the pool alive and returns the pinned slab when numpy lets go
  std::shared_ptr<PoolHandle> pool;
  void* slab;
  SlabLease(std::shared_ptr<PoolHandle> p, void* s) : pool(std::move(p)), slab(s) {}
  SlabLease(const SlabLease&) = delete;
  SlabLease& operator=(const SlabLease&) = delete;
  ~SlabLease() {
    if (pool && pool->p && slab) epb_release_slab(pool->p, slab);
  }
};

class PoolBase {
 public:
  std::shared_ptr<PoolHandle> h;
  std::vector<epb_key_info> keys;
  std::vector<int> key_players;  // epb_state_key_players of each state key
  int players = 1;               // players per env (max_num_players)
  epb_key_info act{};
  std::vector<int32_t> env_seed;
  int device_ordinal = 0;  // resolved CUDA device of the pool

  void Create(const SpecBase& spec, int device, const std::string& precision,
              int env_id_offset) {
    players = spec.desc->players;
    if (players > 1) {
      if (spec.cfg<int>("max_num_players") != players)
        throw std::invalid_argument(std::string(spec.desc->name) + " is a " +
                                    (players == 2 ? "two" : std::to_string(players)) +
                                    "-player game: max_num_players must be " +
                                    std::to_string(players));
    } else if (spec.cfg<int>("max_num_players") != 1) {
      throw std::invalid_argument("max_num_players != 1 is outside the accelerated path");
    }
    if (spec.desc->kind == EPB_HALF_CHEETAH) {
      // post_constraint (v5) only adds mj_rnePostConstraint (mujoco_env.h:145-147), whose
      // outputs (cacc/cfrc_*) HalfCheetah never reads: accepted, no effect on any column.
      if (spec.cfg<int>("frame_stack") != 1)
        throw std::invalid_argument("HalfCheetah: frame_stack != 1 is not accelerated");
      if (!spec.cfg<bool>("exclude_current_positions_from_observation"))
        throw std::invalid_argument(
            "HalfCheetah: exclude_current_positions_from_observation=False is not accelerated");
      // the reference takes frame_skip substeps and divides by dt = frame_skip * timestep
      // (half_cheetah.h:151-152): no substep and a NaN reward at 0, nonsense below
      if (spec.cfg<int>("frame_skip") < 1)
        throw std::invalid_argument("HalfCheetah: frame_skip must be >= 1 (the reward divides "
                                    "by dt = frame_skip * timestep)");
    }
    epb_config c{};
    c.num_envs = spec.cfg<int>("num_envs");
    c.batch_size = spec.cfg<int>("batch_size");
    c.seed = spec.cfg<int>("seed");
    env_seed.clear();
    for (int s : spec.cfg<std::vector<int>>("env_seed")) env_seed.push_back(s);
    if (!env_seed.empty() && static_cast<int>(env_seed.size()) != c.num_envs)
      throw std::invalid_argument("`env_seed` must contain exactly one seed for each env");
    c.env_seed = env_seed.empty() ? nullptr : env_seed.data();
    c.max_episode_steps = spec.cfg<int>("max_episode_steps");
    c.env_id_offset = 0;
    c.device = 0;
    c.precision = EPB_PREC_F64;
    c.iopt = -1;
    c.frame_skip = 0;
    c.ctrl_cost_weight = c.forward_reward_weight = c.reset_noise_scale = std::nan("");
    switch (spec.desc->kind) {
      case EPB_PENDULUM: c.iopt = spec.cfg<int>("version"); break;
      case EPB_FROZEN_LAKE: c.iopt = spec.cfg<int>("size"); break;
      case EPB_CLIFF_WALKING: c.iopt = spec.cfg<bool>("is_slippery") ? 1 : 0; break;
      case EPB_BLACKJACK:
        c.iopt = (spec.cfg<bool>("natural") ? 1 : 0) | (spec.cfg<bool>("sab") ? 2 : 0);
        break;
      case EPB_GAME2048: c.iopt = spec.cfg<bool>("game2048_add_random_cell") ? 1 : 0; break;
      case EPB_HALF_CHEETAH:  // verbatim: any sign, as the reference (half_cheetah.h:89-95)
        c.frame_skip = spec.cfg<int>("frame_skip");
        c.ctrl_cost_weight = spec.cfg<double>("ctrl_cost_weight");
        c.forward_reward_weight = spec.cfg<double>("forward_reward_weight");
        c.reset_noise_scale = spec.cfg<double>("reset_noise_scale");
        break;
      default: break;
    }
    // Engine extensions (not part of the reference config tuple): optional ctor kwargs, or
    // environment variables so the reference's own Python layer -- which only forwards
    // the config tuple -- can still select them.
    std::string prec = precision;
    if (device < 0) {
      const char* d = std::getenv("ENVPOOL_B200_DEVICE");
      device = d ? std::atoi(d) : 0;
    }
    if (prec.empty()) {
      const char* pr = std::getenv("ENVPOOL_B200_PRECISION");
      prec = pr ? pr : "f64";
    }
    if (env_id_offset < 0) {
      const char* o = std::getenv("ENVPOOL_B200_ENV_ID_OFFSET");
      env_id_offset = o ? std::atoi(o) : 0;
    }
    if (prec != "f64" && prec != "f32")
      throw std::invalid_argument("precision must be 'f64' or 'f32'");
    c.device = device;
    device_ordinal = device;
    c.precision = prec == "f32" ? EPB_PREC_F32 : EPB_PREC_F64;
    c.env_id_offset = env_id_offset;
    h = std::make_shared<PoolHandle>();
    check(epb_create(spec.engine_kind(), &c, &h->p));
    if (spec.desc->kind == EPB_GO_19X19)
      check(epb_go_config(h->p, spec.cfg<double>("komi"), spec.cfg<int>("max_terminal_steps")));
    if (!spec.game2048_initial.empty() || !spec.game2048_replay.empty())
      check(epb_game2048_boards(
          h->p, spec.game2048_initial.empty() ? nullptr : spec.game2048_initial.data(),
          spec.game2048_replay.empty() ? nullptr : spec.game2048_replay.data()));
    const MinesweeperConfig& ms = spec.minesweeper;
    if (!ms.mines.empty() || ms.replay)
      check(epb_minesweeper_config(h->p, ms.mines.empty() ? nullptr : ms.mines.data(),
                                   ms.replay ? ms.boards.data() : nullptr,
                                   ms.replay ? ms.rewards.data() : nullptr,
                                   ms.replay ? ms.done.data() : nullptr));
    keys.resize(epb_num_state_keys(h->p));
    key_players.resize(keys.size());
    for (size_t k = 0; k < keys.size(); ++k) {
      check(epb_state_key(h->p, (int)k, &keys[k]));
      key_players[k] = epb_state_key_players(h->p, (int)k);
      if (key_players[k] < 1) check(key_players[k]);
    }
    check(epb_action_key(h->p, &act));
  }

  // Multi-player pools: the action row of each env row is the one of its first player row, the
  // first i with players.env_id[i] == env_id (Env::ParseAction, core/env.h:146-176, and the
  // `action["action"_][0]` each game's Step reads).  An env without a player row raises.
  py::array_t<int, py::array::c_style> FirstPlayerActions(
      const py::array_t<int, py::array::c_style | py::array::forcecast>& ids,
      const py::array& player_env_id, const py::array& action) const {
    py::array_t<int, py::array::c_style | py::array::forcecast> pids(player_env_id);
    py::array_t<int, py::array::c_style | py::array::forcecast> pa(action);
    const int m = static_cast<int>(pids.size());
    if (static_cast<int64_t>(pa.nbytes()) != static_cast<int64_t>(m) * act.row_bytes)
      throw std::invalid_argument("action batch does not match players.env_id batch");
    const int num_envs = epb_num_envs(h->p);
    std::vector<int> first(num_envs, -1);
    const int* pid = pids.data();
    for (int i = m - 1; i >= 0; --i)
      if (pid[i] >= 0 && pid[i] < num_envs) first[pid[i]] = i;
    const int n = static_cast<int>(ids.size());
    py::array_t<int, py::array::c_style> out(n);
    int* o = out.mutable_data();
    const int* id = ids.data();
    const int* av = pa.data();
    for (int i = 0; i < n; ++i) {
      const int e = id[i];
      if (e < 0 || e >= num_envs)
        throw std::invalid_argument("env_id " + std::to_string(e) + " out of range");
      if (first[e] < 0)
        throw std::invalid_argument("env_id " + std::to_string(e) +
                                    " has no row in players.env_id: no action for that env");
      o[i] = av[first[e]];
    }
    return out;
  }

  // PyEnvPool::PySend, py_envpool.h:244-250
  void Send(const std::vector<py::array>& action) {
    if (action.size() != 3) throw std::invalid_argument("expected [env_id, players.env_id, action]");
    py::array_t<int, py::array::c_style | py::array::forcecast> ids(action[0]);
    py::array a;
    if (players > 1) a = FirstPlayerActions(ids, action[1], action[2]);
    else if (act.dtype == EPB_I32) a = py::array_t<int, py::array::c_style | py::array::forcecast>(action[2]);
    else if (act.dtype == EPB_F32) a = py::array_t<float, py::array::c_style | py::array::forcecast>(action[2]);
    else a = py::array_t<double, py::array::c_style | py::array::forcecast>(action[2]);
    int n = static_cast<int>(ids.size());
    if (static_cast<int64_t>(a.nbytes()) != static_cast<int64_t>(n) * act.row_bytes)
      throw std::invalid_argument("action batch does not match env_id batch");
    const void* ap = a.data();
    const int32_t* ip = ids.data();
    int rc;
    {
      py::gil_scoped_release release;
      rc = epb_send(h->p, ap, ip, n);
    }
    check(rc);
  }

  // PyEnvPool::PyRecv, py_envpool.h:255-266: zero-copy numpy views over one pinned slab;
  // a capsule keeps the slab (and the pool) alive until every returned array is dropped.
  // A per-player column comes back as [n * P, ...], the reference's player rows: the engine
  // keeps the P rows of an env row next to each other.
  std::vector<py::array> Recv() {
    void* slab = nullptr;
    int n = 0, row0 = 0, rc;
    {
      py::gil_scoped_release release;
      rc = epb_recv_slab_ex(h->p, &slab, &row0, &n);
    }
    check(rc);
    auto lease = std::make_shared<SlabLease>(h, slab);
    std::vector<py::array> ret;
    ret.reserve(keys.size());
    for (size_t kk = 0; kk < keys.size(); ++kk) {
      const epb_key_info& k = keys[kk];
      const int P = key_players[kk];
      auto* holder = new std::shared_ptr<SlabLease>(lease);
      py::capsule cap(holder, [](void* p) { delete static_cast<std::shared_ptr<SlabLease>*>(p); });
      std::vector<py::ssize_t> shape = {static_cast<py::ssize_t>(n) * P};
      for (int i = 0; i < k.ndim; ++i) shape.push_back(k.shape[i]);
      char* base = static_cast<char*>(slab) + k.slab_offset +
                   static_cast<size_t>(row0) * k.row_bytes;
      switch (k.dtype) {
        case EPB_I32: ret.emplace_back(py::array(shape, reinterpret_cast<int*>(base), cap)); break;
        case EPB_F32: ret.emplace_back(py::array(shape, reinterpret_cast<float*>(base), cap)); break;
        case EPB_F64: ret.emplace_back(py::array(shape, reinterpret_cast<double*>(base), cap)); break;
        default: ret.emplace_back(py::array(shape, reinterpret_cast<bool*>(base), cap)); break;
      }
    }
    return ret;
  }

  // PyEnvPool::PyReset, py_envpool.h:271-276
  void Reset(const py::array& env_ids) {
    py::array_t<int, py::array::c_style | py::array::forcecast> ids(env_ids);
    const int32_t* ip = ids.data();
    int n = static_cast<int>(ids.size()), rc;
    {
      py::gil_scoped_release release;
      rc = epb_reset(h->p, ip, n);
    }
    check(rc);
  }
  py::array Render(const py::array&, int, int, int) {
    throw std::runtime_error("render not implemented for this environment");
  }
  py::tuple Xla() { throw std::runtime_error("XLA is not available in envpool_b200"); }
  std::uintptr_t Handle() const { return reinterpret_cast<std::uintptr_t>(h->p); }
  int Device() const { return device_ordinal; }
};

// One distinct C++ type per env so pybind11 creates one distinct Python class each.
template <int K>
struct Tag {
  static const EnvDesc* desc;
};
template <int K>
const EnvDesc* Tag<K>::desc = nullptr;

template <int K>
class PySpec : public SpecBase {
 public:
  explicit PySpec(const py::tuple& conf) : SpecBase(Tag<K>::desc, conf) {}
};
template <int K>
class PyPool : public PoolBase {
 public:
  PySpec<K> py_spec;
  PyPool(const PySpec<K>& s, int device, const std::string& precision, int env_id_offset)
      : py_spec(s) {
    Create(py_spec, device, precision, env_id_offset);
  }
};

template <int K>
void register_env(py::module_& m, const EnvDesc* d) {
  Tag<K>::desc = d;
  std::string stem = d->name;
  py::object abc = py::module_::import("abc").attr("ABCMeta");
  std::vector<std::string> cfg_keys(kCommonKeys, kCommonKeys + kNumCommon);
  for (auto& k : d->cfg_keys) cfg_keys.push_back(k);
  py::tuple defaults = py::tuple(common_defaults() + d->cfg_defaults());
  PySpec<K> probe(defaults);
  auto state_keys = probe.StateKeys();
  auto action_keys = probe.ActionKeys();

  py::class_<PySpec<K>> spec(m, ("_" + stem + "EnvSpec").c_str(), py::metaclass(abc));
  spec.def(py::init<const py::tuple&>())
      .def_readonly("_config_values", &PySpec<K>::config_values)
      .def_property_readonly("_state_spec", [](const PySpec<K>& s) { return s.StateSpecPy(); })
      .def_property_readonly("_action_spec", [](const PySpec<K>& s) { return s.ActionSpecPy(); });
  spec.attr("_state_keys") = state_keys;
  spec.attr("_action_keys") = action_keys;
  spec.attr("_config_keys") = cfg_keys;
  spec.attr("_default_config_values") = defaults;

  py::class_<PyPool<K>> pool(m, ("_" + stem + "EnvPool").c_str(), py::metaclass(abc));
  pool.def(py::init<const PySpec<K>&, int, const std::string&, int>(), py::arg("spec"),
           py::arg("device") = -1, py::arg("precision") = "", py::arg("env_id_offset") = -1)
      .def_readonly("_spec", &PyPool<K>::py_spec)
      .def("_recv", &PyPool<K>::Recv)
      .def("_send", &PyPool<K>::Send)
      .def("_reset", &PyPool<K>::Reset)
      .def("_render", &PyPool<K>::Render)
      .def("_xla", &PyPool<K>::Xla)
      // extension: raw epb_pool* for the device-resident C-ABI entry points
      .def_property_readonly("_handle", &PyPool<K>::Handle)
      .def_property_readonly("_device", &PyPool<K>::Device);
  pool.attr("_state_keys") = state_keys;
  pool.attr("_action_keys") = action_keys;
}

#define DESC(NAME, KIND, KEYS, DEFAULTS)                                   \
  static EnvDesc desc_##NAME{#NAME, KIND, KEYS, []() -> py::tuple DEFAULTS}
// a kind with more than one player per env
#define DESC_PLAYERS(NAME, KIND, PLAYERS, KEYS, DEFAULTS)                  \
  static EnvDesc desc_##NAME{#NAME, KIND, KEYS, []() -> py::tuple DEFAULTS, PLAYERS}

using S = std::vector<std::string>;

}  // namespace

#ifndef EPB_MODULE_NAME
#error "EPB_MODULE_NAME must be defined"
#endif

PYBIND11_MODULE(EPB_MODULE_NAME, m) {
  m.attr("__engine__") = "envpool_b200";
  m.attr("__abi_version__") = epb_abi_version();
#if defined(EPB_FAMILY_CLASSIC_CONTROL)
  // classic_control/classic_control.cc:30-45
  DESC(CartPole, EPB_CARTPOLE, S{"reward_threshold"}, { return py::make_tuple(195.0); });
  DESC(Pendulum, EPB_PENDULUM, S{"version"}, { return py::make_tuple(0); });
  DESC(MountainCar, EPB_MOUNTAIN_CAR, S{"reward_threshold"}, { return py::make_tuple(-110.0); });
  DESC(MountainCarContinuous, EPB_MOUNTAIN_CAR_CONTINUOUS, S{"reward_threshold"},
       { return py::make_tuple(90.0); });
  DESC(Acrobot, EPB_ACROBOT, S{"reward_threshold"}, { return py::make_tuple(-100.0); });
  register_env<EPB_CARTPOLE>(m, &desc_CartPole);
  register_env<EPB_PENDULUM>(m, &desc_Pendulum);
  register_env<EPB_MOUNTAIN_CAR>(m, &desc_MountainCar);
  register_env<EPB_MOUNTAIN_CAR_CONTINUOUS>(m, &desc_MountainCarContinuous);
  register_env<EPB_ACROBOT>(m, &desc_Acrobot);
#elif defined(EPB_FAMILY_TOY_TEXT)
  // toy_text/toy_text.cc:33-48
  DESC(Catch, EPB_CATCH, (S{"height", "width"}), { return py::make_tuple(10, 5); });
  DESC(FrozenLake, EPB_FROZEN_LAKE, (S{"reward_threshold", "size"}),
       { return py::make_tuple(0.7, 4); });
  DESC(Taxi, EPB_TAXI, S{"reward_threshold"}, { return py::make_tuple(8.0); });
  DESC(NChain, EPB_NCHAIN, S{}, { return py::tuple(); });
  DESC(CliffWalking, EPB_CLIFF_WALKING, S{"is_slippery"}, { return py::make_tuple(false); });
  DESC(Blackjack, EPB_BLACKJACK, (S{"natural", "sab"}), { return py::make_tuple(false, true); });
  register_env<EPB_CATCH>(m, &desc_Catch);
  register_env<EPB_FROZEN_LAKE>(m, &desc_FrozenLake);
  register_env<EPB_TAXI>(m, &desc_Taxi);
  register_env<EPB_NCHAIN>(m, &desc_NChain);
  register_env<EPB_CLIFF_WALKING>(m, &desc_CliffWalking);
  register_env<EPB_BLACKJACK>(m, &desc_Blackjack);
#elif defined(EPB_FAMILY_JUMANJI)
  // jumanji/jumanji_envpool.cc (Game2048 and Minesweeper)
  DESC(Game2048, EPB_GAME2048,
       (S{"game2048_initial_board", "game2048_replay_boards", "game2048_add_random_cell"}),
       { return py::make_tuple(std::string(""), std::string(""), true); });
  DESC(Minesweeper, EPB_MINESWEEPER,
       (S{"minesweeper_mine_locations", "minesweeper_replay_boards", "minesweeper_replay_rewards",
          "minesweeper_replay_done"}),
       {
         return py::make_tuple(std::string(""), std::string(""), std::string(""),
                               std::string(""));
       });
  register_env<EPB_GAME2048>(m, &desc_Game2048);
  register_env<EPB_MINESWEEPER>(m, &desc_Minesweeper);
#elif defined(EPB_FAMILY_MUJOCO_GYM)
  // mujoco/gym/mujoco_envpool.cc (HalfCheetah only: the one MuJoCo task on the hot path)
  DESC(GymHalfCheetah, EPB_HALF_CHEETAH,
       (S{"reward_threshold", "frame_skip", "frame_stack", "post_constraint",
          "exclude_current_positions_from_observation", "xml_file",
          "gymnasium_v5_render_camera", "ctrl_cost_weight", "forward_reward_weight",
          "reset_noise_scale"}),
       {
         return py::make_tuple(4800.0, 5, 1, true, true, std::string("half_cheetah.xml"),
                               false, 0.1, 1.0, 0.1);
       });
  register_env<EPB_HALF_CHEETAH>(m, &desc_GymHalfCheetah);
#elif defined(EPB_FAMILY_PGX)
  // pgx/pgx.cc (TicTacToe, ConnectFour, Hex, Othello, Go and the chess games: the two-player board
  // games on the
  // hot path)
  DESC_PLAYERS(TicTacToe, EPB_TIC_TAC_TOE, 2, S{"task"},
               { return py::make_tuple(std::string("tic_tac_toe")); });
  DESC_PLAYERS(ConnectFour, EPB_CONNECT_FOUR, 2, S{"task"},
               { return py::make_tuple(std::string("connect_four")); });
  DESC_PLAYERS(Hex, EPB_HEX, 2, S{"task"}, { return py::make_tuple(std::string("hex")); });
  DESC_PLAYERS(Othello, EPB_OTHELLO, 2, S{"task"},
               { return py::make_tuple(std::string("othello")); });
  register_env<EPB_TIC_TAC_TOE>(m, &desc_TicTacToe);
  register_env<EPB_CONNECT_FOUR>(m, &desc_ConnectFour);
  register_env<EPB_HEX>(m, &desc_Hex);
  register_env<EPB_OTHELLO>(m, &desc_Othello);
  // pgx/go.h: one class for the three boards, as the reference's GoEnvSpec / GoEnvPool
  DESC_PLAYERS(Go, EPB_GO_19X19, 2,
               (S{"board_size", "komi", "history_length", "max_terminal_steps", "rules", "task"}),
               {
                 return py::make_tuple(19, 7.5, 8, 0, std::string("pgx"),
                                       std::string("go_19x19"));
               });
  register_env<EPB_GO_19X19>(m, &desc_Go);
  // pgx/chess_games.h
  DESC_PLAYERS(Chess, EPB_CHESS, 2, S{"task"}, { return py::make_tuple(std::string("chess")); });
  DESC_PLAYERS(GardnerChess, EPB_GARDNER_CHESS, 2, S{"task"},
               { return py::make_tuple(std::string("gardner_chess")); });
  register_env<EPB_CHESS>(m, &desc_Chess);
  register_env<EPB_GARDNER_CHESS>(m, &desc_GardnerChess);
#else
#error "define one EPB_FAMILY_* macro"
#endif
}
