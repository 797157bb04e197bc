"""TEST INFRASTRUCTURE ONLY: ctypes wrapper over oracle/libep_oracle.so (ep_oracle.c).

The product package envpool_b200 never imports this module; only tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / reference legs do.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_SO = os.path.join(_HERE, "libep_oracle.so")

KINDS = {
    "CartPole": 0, "Pendulum": 1, "Acrobot": 2, "MountainCar": 3,
    "MountainCarContinuous": 4, "FrozenLake": 5, "Catch": 6, "Taxi": 7,
    "NChain": 8, "CliffWalking": 9, "Blackjack": 10, "HalfCheetah": 11,
}
_DT = {("done",): np.bool_, ("trunc",): np.bool_}


def build(force: bool = False) -> str:
    srcs = [os.path.join(_HERE, f) for f in
            ("ep_oracle.c", "ep_oracle.h", "mjc_oracle.c", "mjc_oracle.h")]
    if (force or not os.path.exists(ORACLE_SO) or
            any(os.path.getmtime(s) > os.path.getmtime(ORACLE_SO) for s in srcs)):
        subprocess.check_call(["make", "-C", _HERE, "oracle"],
                              stdout=subprocess.DEVNULL)
    return ORACLE_SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = ctypes.CDLL(build())
        vp, ci = ctypes.c_void_p, ctypes.c_int
        L.epo_create.restype = vp
        cd = ctypes.c_double
        L.epo_create.argtypes = [ci, ci, ci, vp, ci, ci, ci, cd, cd, cd]
        L.epo_destroy.argtypes = [vp]
        L.epo_reset.argtypes = [vp, vp, ci]
        L.epo_step.argtypes = [vp, vp, vp, ci]
        L.epo_num_keys.argtypes = [vp]
        L.epo_key_name.restype = ctypes.c_char_p
        L.epo_key_name.argtypes = [vp, ci]
        L.epo_key_elem_size.argtypes = [vp, ci]
        L.epo_key_row_elems.argtypes = [vp, ci]
        L.epo_key_data.restype = vp
        L.epo_key_data.argtypes = [vp, ci]
        L.epo_action_elem_size.argtypes = [vp]
        L.epo_action_row_elems.argtypes = [vp]
        L.epo_get_state.argtypes = [vp, ci, vp, vp, vp]
        L.epo_set_state.argtypes = [vp, ci, vp, ci, ci]
        L.epo_get_states.argtypes = [vp, vp]
        L.epo_mjc_set.argtypes = [vp, ci, vp, ci, ci]
        L.epo_mjc_get.argtypes = [vp, ci, vp]
        L.epo_debug_draw.restype = ctypes.c_uint32
        L.epo_debug_draw.argtypes = [vp, ci]
        L.epo_debug_set_rng.argtypes = [vp, ci, vp, ci]
        L.epo_debug_get_rng.argtypes = [vp, ci, vp, vp]
        L.epo_set_int_states.argtypes = [vp] * 8
        L.epo_get_int_states.argtypes = [vp] * 8
        L.epo_trig.argtypes = [ci, vp, ci, vp, vp]
        _lib = L
    return _lib


def libm_trig(x, want_sin=True, want_cos=True):
    """libm's sin and cos of every element of `x` (float64: sin / cos, float32: sinf / cosf),
    the functions the oracle's classic_control steps call; (sin, cos), None where not wanted.
    numpy's own sin is not libm's, so the oracle's values come from here."""
    x = np.ascontiguousarray(x)
    kind = {np.dtype(np.float64): 0, np.dtype(np.float32): 1}[x.dtype]
    s = np.empty_like(x) if want_sin else None
    c = np.empty_like(x) if want_cos else None
    rc = lib().epo_trig(kind, x.ctypes.data, x.size, None if s is None else s.ctypes.data,
                        None if c is None else c.ctypes.data)
    assert rc == 0, rc
    return s, c


def _key_dtype(name, elem_size, kind):
    if name in ("done", "trunc"):
        return np.bool_
    if elem_size == 8:
        return np.float64
    int_obs = kind in (5, 7, 8, 9, 10)
    if name in ("reward", "discount", "info:prob", "info:state"):
        return np.float32
    if name == "obs":
        return np.int32 if int_obs else np.float32
    return np.int32


class OraclePool:
    """CPU restatement of AsyncEnvPool<Env> in sync mode.  The four HalfCheetah options are
    used as given, with the reference's defaults (half_cheetah.h:32-42)."""

    def __init__(self, task, num_envs, seed=42, max_episode_steps=-1, iopt=-1,
                 env_seed=None, frame_skip=5, ctrl_cost_weight=0.1, forward_reward_weight=1.0,
                 reset_noise_scale=0.1):
        self.kind = KINDS[task]
        self.n = num_envs
        es = None
        if env_seed is not None:
            self._env_seed = np.ascontiguousarray(env_seed, dtype=np.int32)
            es = self._env_seed.ctypes.data
        self.h = lib().epo_create(self.kind, num_envs, seed, es, max_episode_steps, iopt,
                                  frame_skip, ctrl_cost_weight, forward_reward_weight,
                                  reset_noise_scale)
        if not self.h:
            raise RuntimeError(f"epo_create({task}) failed")
        L = lib()
        self.keys = []
        for k in range(L.epo_num_keys(self.h)):
            name = L.epo_key_name(self.h, k).decode()
            es_ = L.epo_key_elem_size(self.h, k)
            self.keys.append((name, _key_dtype(name, es_, self.kind),
                              L.epo_key_row_elems(self.h, k)))
        self.act_dtype = (np.float64 if L.epo_action_elem_size(self.h) == 8 else
                          np.float32 if self.kind in (1, 4) else np.int32)
        self.act_row = L.epo_action_row_elems(self.h)

    def close(self):
        if self.h:
            lib().epo_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def _collect(self, n):
        out = {}
        for k, (name, dt, row) in enumerate(self.keys):
            ptr = lib().epo_key_data(self.h, k)
            nbytes = n * row * np.dtype(dt).itemsize
            buf = (ctypes.c_char * nbytes).from_address(ptr)
            arr = np.frombuffer(buf, dtype=dt).copy()
            if name == "obs" and self.kind == 6:
                arr = arr.reshape(n, 10, 5)
            elif row > 1:
                arr = arr.reshape(n, row)
            out[name] = arr
        return out

    def reset(self, env_ids=None):
        if env_ids is None:
            lib().epo_reset(self.h, None, self.n)
            return self._collect(self.n)
        ids = np.ascontiguousarray(env_ids, dtype=np.int32)
        lib().epo_reset(self.h, ids.ctypes.data, len(ids))
        return self._collect(len(ids))

    def step(self, action, env_ids=None):
        a = np.ascontiguousarray(action, dtype=self.act_dtype)
        if env_ids is None:
            lib().epo_step(self.h, a.ctypes.data, None, self.n)
            return self._collect(self.n)
        ids = np.ascontiguousarray(env_ids, dtype=np.int32)
        lib().epo_step(self.h, a.ctypes.data, ids.ctypes.data, len(ids))
        return self._collect(len(ids))

    def set_state(self, eid, s5, done, cur):
        buf = (ctypes.c_double * 5)(*[float(x) for x in s5])
        lib().epo_set_state(self.h, eid, buf, int(done), int(cur))

    def get_state(self, eid):
        buf = (ctypes.c_double * 5)()
        d, c = ctypes.c_int(), ctypes.c_int()
        lib().epo_get_state(self.h, eid, buf, ctypes.byref(d), ctypes.byref(c))
        return list(buf), d.value, c.value

    def states(self):
        """[num_envs, 5] continuous state s[0..4] of every env."""
        out = np.zeros((self.n, 5))
        lib().epo_get_states(self.h, out.ctypes.data)
        return out

    def set_int_states(self, st):
        """toy_text: overwrite every env's integer state at once, RNG untouched.  `st` is a
        dict of int32 arrays as int_states() returns: i [N, 8], done [N], cur [N] and, for
        Blackjack, player / dealer [N, 32] with nplayer / ndealer [N]."""
        a = {k: np.ascontiguousarray(v, dtype=np.int32) for k, v in st.items()}
        assert a["i"].shape == (self.n, 8) and a["done"].shape == a["cur"].shape == (self.n,)
        hands = "player" in a
        if hands:
            assert a["player"].shape == a["dealer"].shape == (self.n, 32)
        ptr = lambda k: a[k].ctypes.data if k in a else None  # noqa: E731
        lib().epo_set_int_states(self.h, ptr("i"), ptr("player"), ptr("nplayer"),
                                 ptr("dealer"), ptr("ndealer"), ptr("done"), ptr("cur"))

    def int_states(self):
        """Every env's integer state, done flag and step counter (the layout set_int_states
        takes); Blackjack's hands too."""
        n = self.n
        st = {"i": np.zeros((n, 8), np.int32), "done": np.zeros(n, np.int32),
              "cur": np.zeros(n, np.int32)}
        if self.kind == KINDS["Blackjack"]:
            st.update(player=np.zeros((n, 32), np.int32), dealer=np.zeros((n, 32), np.int32),
                      nplayer=np.zeros(n, np.int32), ndealer=np.zeros(n, np.int32))
        ptr = lambda k: st[k].ctypes.data if k in st else None  # noqa: E731
        lib().epo_get_int_states(self.h, ptr("i"), ptr("player"), ptr("nplayer"),
                                 ptr("dealer"), ptr("ndealer"), ptr("done"), ptr("cur"))
        return st

    def set_rng(self, eid, mt624, idx):
        """Load env `eid`'s std::mt19937: 624 table words and the read position (624 = the
        next draw regenerates the table)."""
        row = np.ascontiguousarray(mt624, dtype=np.uint32)
        assert row.shape == (624,)
        lib().epo_debug_set_rng(self.h, eid, row.ctypes.data, int(idx))

    def rng(self, eid):
        mt, idx = np.zeros(624, np.uint32), ctypes.c_int()
        lib().epo_debug_get_rng(self.h, eid, mt.ctypes.data, ctypes.byref(idx))
        return mt, idx.value

    def mjc_set(self, eid, s27, done, cur):
        buf = np.ascontiguousarray(s27, dtype=np.float64)
        lib().epo_mjc_set(self.h, eid, buf.ctypes.data, int(done), int(cur))

    def mjc_get(self, eid):
        buf = np.zeros(27)
        lib().epo_mjc_get(self.h, eid, buf.ctypes.data)
        return buf

    def draw(self, eid):
        return lib().epo_debug_draw(self.h, eid)


class MjcSim:
    """Direct handle on the HalfCheetah physics restatement (oracle/mjc_oracle.c)."""

    def __init__(self):
        L = lib()
        vp = ctypes.c_void_p
        L.mjc_make_half_cheetah.restype = vp
        L.mjc_make_data.restype = vp
        L.mjc_make_data.argtypes = [vp]
        L.mjc_free_model.argtypes = [vp]
        L.mjc_free_data.argtypes = [vp]
        L.mjc_qpos_mut.restype = ctypes.POINTER(ctypes.c_double)
        L.mjc_qpos_mut.argtypes = [vp]
        L.mjc_qvel_mut.restype = ctypes.POINTER(ctypes.c_double)
        L.mjc_qvel_mut.argtypes = [vp]
        L.mjc_step.argtypes = [vp, vp, vp, ctypes.c_int]
        L.mjc_forward.argtypes = [vp, vp]
        L.mjc_nefc.argtypes = [vp]
        L.mjc_model_constants.argtypes = [vp, vp, ctypes.c_int]
        L.mjc_debug_dynamics.restype = ctypes.c_double
        L.mjc_debug_dynamics.argtypes = [vp, vp, vp, vp, vp]
        self.L = L
        self.m = L.mjc_make_half_cheetah()
        self.d = L.mjc_make_data(self.m)

    def close(self):
        if self.d:
            self.L.mjc_free_data(self.d)
            self.L.mjc_free_model(self.m)
            self.d = self.m = None

    def __del__(self):
        self.close()

    @property
    def qpos(self):
        return np.ctypeslib.as_array(self.L.mjc_qpos_mut(self.d), shape=(9,))

    @property
    def qvel(self):
        return np.ctypeslib.as_array(self.L.mjc_qvel_mut(self.d), shape=(9,))

    def step(self, action, frame_skip=1):
        a = np.ascontiguousarray(action, dtype=np.float64)
        self.L.mjc_step(self.m, self.d, a.ctypes.data, frame_skip)

    def forward(self):
        self.L.mjc_forward(self.m, self.d)

    @property
    def nefc(self):
        return self.L.mjc_nefc(self.d)

    def dynamics(self, qpos, qvel):
        """(M [9,9], bias [9], gravitational potential) at an arbitrary (qpos, qvel)."""
        q = np.ascontiguousarray(qpos, dtype=np.float64)
        v = np.ascontiguousarray(qvel, dtype=np.float64)
        M, c = np.zeros((9, 9)), np.zeros(9)
        V = self.L.mjc_debug_dynamics(self.m, q.ctypes.data, v.ctypes.data, M.ctypes.data,
                                      c.ctypes.data)
        return M, c, V

    def solve_problem(self):
        """Runs the forward dynamics of the current state and returns the constraint problem as
        the solver sees it plus its answer: dict(M, qfrc_smooth, J, D, aref, qacc)."""
        vp = ctypes.c_void_p
        self.L.mjc_debug_solve.argtypes = [vp, vp, vp, vp, vp, vp, vp, ctypes.c_int, vp]
        cap = 80
        M, fs, qacc = np.zeros((9, 9)), np.zeros(9), np.zeros(9)
        J, D, aref = np.zeros((cap, 9)), np.zeros(cap), np.zeros(cap)
        n = self.L.mjc_debug_solve(self.m, self.d, M.ctypes.data, fs.ctypes.data, J.ctypes.data,
                                   D.ctypes.data, aref.ctypes.data, cap, qacc.ctypes.data)
        return {"M": M, "qfrc_smooth": fs, "J": J[:n].copy(), "D": D[:n].copy(),
                "aref": aref[:n].copy(), "qacc": qacc}

    def constants(self):
        buf = np.zeros(64)
        n = self.L.mjc_model_constants(self.m, buf.ctypes.data, 64)
        c = buf[:n]
        return {"mass": c[0:28:4].copy(), "com": np.stack([c[1:28:4], c[2:28:4]], 1),
                "iyy": c[3:28:4].copy(), "dof_invweight0": c[28:37].copy(),
                "body_invweight0": c[37:51].reshape(7, 2).copy(), "meaninertia": c[51]}
