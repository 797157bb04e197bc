"""Shared helpers for the parity tests (test infrastructure; may import oracle/)."""
import glob
import json
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")

EXACT_KEYS = ("info:env_id", "info:players.env_id", "elapsed_step", "done", "discount",
              "step_type", "trunc")
INT_TASKS = ("FrozenLake", "Catch", "Taxi", "NChain", "CliffWalking", "Blackjack")
N_ACT = {"CartPole": 2, "Acrobot": 3, "MountainCar": 3, "FrozenLake": 4, "Catch": 3,
         "Taxi": 6, "NChain": 2, "CliffWalking": 4, "Blackjack": 2}
# registered max_episode_steps (envpool/*/registration.py) and default iopt per task
REGISTERED = {
    "CartPole": (500, -1), "Pendulum": (200, 1), "Acrobot": (500, -1),
    "MountainCar": (200, -1), "MountainCarContinuous": (999, -1),
    "FrozenLake": (100, 4), "Catch": (-1, -1), "Taxi": (200, -1), "NChain": (1000, -1),
    "CliffWalking": (-1, 0), "Blackjack": (-1, 2),
}


def golden_cases():
    return sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "*.npz")))


def load_golden(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = json.loads(str(z["meta"]))
    data = {k: z[k] for k in z.files if k != "meta"}
    return meta, data


def random_actions(task, rng, shape_prefix, act_dtype=None):
    if task in ("Pendulum", "MountainCarContinuous"):
        return rng.uniform(-2.5, 2.5, size=tuple(shape_prefix) + (1,)).astype(np.float32)
    if task == "HalfCheetah":
        return rng.uniform(-1.0, 1.0, size=tuple(shape_prefix) + (6,)).astype(np.float64)
    return rng.integers(0, N_ACT[task], size=tuple(shape_prefix)).astype(np.int32)


def row_tolerance(task, float_atol, elapsed):
    """Per-row float tolerance for FREE-RUNNING trajectory comparisons.  Acrobot is a
    chaotic double pendulum: the <= 2 ulp difference between CUDA's and glibc's double
    sin/cos (1e-16) is amplified along an episode (measured 1.5e-6 after 400 steps), so its
    free-running tolerance opens with the depth into the episode.  Its per-step arithmetic
    is pinned separately, without amplification, by the teacher-forced test
    (test_gpu_parity.py::test_teacher_forced_single_step).  Every other env keeps
    float_atol for the whole episode."""
    tol = np.full(elapsed.shape, float_atol, dtype=np.float64)
    if task == "Acrobot" and float_atol > 0:
        tol = np.where(elapsed > 300, 5e-2, np.where(elapsed > 150, 1e-4, float_atol))
    return tol


def assert_batch_equal(got, want, task, float_atol=0.0, ctx=""):
    """Integer/bool/flag columns bit-exact; float columns within float_atol (0 = exact),
    relative-absolute: |err| <= tol * (1 + |ref|)."""
    row_tol = row_tolerance(task, float_atol, want["elapsed_step"])
    for k, w in want.items():
        g = got[k]
        assert g.shape == w.shape, (ctx, k, g.shape, w.shape)
        assert g.dtype == w.dtype, (ctx, k, g.dtype, w.dtype)
        if g.dtype.kind in "ib" or k in EXACT_KEYS or task in INT_TASKS or float_atol == 0.0:
            if not np.array_equal(g, w):
                bad = np.argwhere(np.asarray(g != w))[:5]
                raise AssertionError(f"{ctx} key {k}: mismatch at {bad.tolist()} "
                                     f"got {g[tuple(bad[0])]} want {w[tuple(bad[0])]}")
        else:
            err = np.abs(g.astype(np.float64) - w.astype(np.float64))
            rt = row_tol.reshape((-1,) + (1,) * (w.ndim - 1))
            tol = rt * (1.0 + np.abs(w.astype(np.float64)))
            if not np.all(err <= tol):
                i = np.unravel_index(np.argmax(err - tol), err.shape)
                raise AssertionError(f"{ctx} key {k}: |err|={err[i]:.3e} > tol at {i} "
                                     f"got {g[i]} want {w[i]}")


# HalfCheetah's task options (half_cheetah.h:32-42).  A table rather than a product: every value
# below appears in at least one row, and the first row is the reference default.
#   frame_skip            1, 2, 5, 7
#   forward_reward_weight 1.0, 0.0, -1.0, 2.5, -0.0
#   ctrl_cost_weight      0.1, 0.0, -0.05, 1e-3
#   reset_noise_scale     0.1, 0.0, 1.0, -0.1   (1.0 starts joints past their limits and the
#                                                torso in the floor: constraint rows from step 1)
HC_OPTIONS = [
    dict(frame_skip=5, forward_reward_weight=1.0, ctrl_cost_weight=0.1, reset_noise_scale=0.1),
    dict(frame_skip=1, forward_reward_weight=0.0, ctrl_cost_weight=0.0, reset_noise_scale=0.0),
    dict(frame_skip=2, forward_reward_weight=-1.0, ctrl_cost_weight=-0.05, reset_noise_scale=1.0),
    dict(frame_skip=7, forward_reward_weight=2.5, ctrl_cost_weight=1e-3, reset_noise_scale=-0.1),
    dict(frame_skip=1, forward_reward_weight=-0.0, ctrl_cost_weight=1e-3, reset_noise_scale=1.0),
    dict(frame_skip=2, forward_reward_weight=2.5, ctrl_cost_weight=0.0, reset_noise_scale=-0.1),
]
HC_DEFAULT = HC_OPTIONS[0]


def hc_options_id(o):
    return ("fs{frame_skip}-fwd{forward_reward_weight:g}-ctrl{ctrl_cost_weight:g}"
            "-noise{reset_noise_scale:g}").format(**o)


def assert_hc_env_algebra(out, x_before, action, opts, ctx=""):
    """HalfCheetahEnv::Step's env-layer algebra (half_cheetah.h:142-160) bit for bit on every row
    of one step's outputs `out`, from qpos[0] before the step and the raw (unclamped) actions:
        x_velocity  = (x_position - x_before) / (frame_skip * timestep)
        reward_run  = x_velocity * forward_reward_weight
        reward_ctrl = -sum_k (ctrl_cost_weight * a_k) * a_k, from 0.0 in k order
        reward      = float32(reward_run + reward_ctrl)
    Rows that reset instead (elapsed_step 0) carry WriteState(0, 0, 0, 0): reward_run is
    0.0 * forward_reward_weight, so -0.0 for a negative weight.  The engine and numpy do the same
    IEEE operations in the same order, so the bytes (signs of zero included) must agree."""
    fwd, wc = opts["forward_reward_weight"], opts["ctrl_cost_weight"]
    stepped = out["elapsed_step"] > 0
    a = np.asarray(action, dtype=np.float64)
    xv = np.where(stepped, (out["info:x_position"] - x_before) / (opts["frame_skip"] * 0.01), 0.0)
    ctrl = np.zeros(len(a))
    for k in range(a.shape[1]):
        ctrl = ctrl + (wc * a[:, k]) * a[:, k]
    ctrl = np.where(stepped, ctrl, 0.0)
    run = xv * fwd
    want = {"info:x_velocity": xv, "info:reward_run": run, "info:reward_ctrl": -ctrl,
            "reward": np.where(stepped, (run + -ctrl).astype(np.float32), np.float32(0.0)),
            "info:x_position": np.where(stepped, out["info:x_position"], 0.0)}
    for k, w in want.items():
        g = out[k]
        w = np.ascontiguousarray(w, dtype=g.dtype)
        if g.tobytes() != w.tobytes():
            bad = np.nonzero(g.view(np.uint8).reshape(len(g), -1) !=
                             w.view(np.uint8).reshape(len(w), -1))[0][:3]
            raise AssertionError(f"{ctx} {k} at rows {bad.tolist()}: got {g[bad].tolist()} "
                                 f"want {w[bad].tolist()}")
