"""Generates tests/golden/popart_tasks_golden.npz.  Run ONLY where /root/reference exists:
    python tests/golden/make_golden_popart_tasks.py

Multi-task PopArt as K independent reference PopArt modules: the UNMODIFIED popart.py (`PopArt`, compensation
on) over the UNMODIFIED running_statistics.py (`EMAMeanStd`) and common/vtrace.py, loaded over tf_numpy_shim
exactly as make_golden_popart.py loads them (its `_install` is imported, nothing is copied).  Task k has a
PopArt instance of its own and, at every step, sees only the batch columns whose task id is k, composed in the
order of generalized_onpolicy_loss.py:94-133 as make_golden_popart.py composes one task.  A task without
columns in a step is not called and keeps its variables.

K = 3 tasks over B = 12 columns with an uneven mix (6 / 4 / 2 columns), four consecutive steps, the third of
which has no column of task 2; rewards of the tasks differ by orders of magnitude (scales 1, 30, 1000), which is
the workload multi-task PopArt exists for.  Every step stores its inputs, the task ids and each task's state
before and after, so machines without /root/reference replay them (tests/test_popart_tasks.py)."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import tf_numpy_shim  # noqa: E402
from make_golden_popart import _install, _log_softmax  # noqa: E402

K, B, T1, A, STEPS = 3, 12, 11, 6, 4
TASK_IDS = (np.array([0, 1, 0, 2, 0, 1, 0, 1, 0, 2, 1, 0], np.int32),
            np.array([1, 1, 0, 2, 0, 0, 2, 1, 0, 0, 1, 0], np.int32),
            np.array([0, 1, 0, 1, 0, 1, 0, 1, 0, 0, 1, 0], np.int32),   # task 2 absent
            np.array([2, 1, 0, 2, 0, 1, 0, 1, 0, 2, 1, 0], np.int32))
REWARD_SCALE = (1.0, 30.0, 1000.0)


def main():
  tf, popart, rs, vtrace, logged = _install()
  T, raw = tf_numpy_shim.Tensor, tf_numpy_shim._raw
  f32 = np.float32
  out = {}
  rng = np.random.default_rng(31)
  discounting, lambda_, baseline_cost, beta = 0.99, 0.95, 0.5, 3e-2
  out['cfg'] = np.asarray([discounting, lambda_, baseline_cost], f32)
  out['beta'] = np.asarray(beta)
  out['K'] = np.asarray(K)
  tasks = []
  for _ in range(K):
    pa = popart.PopArt(rs.EMAMeanStd(beta))
    pa.init()
    tr = pa.mean_std_tracker
    tasks.append((pa, (tr.first_moment, tr.second_moment, pa.compensation_std, pa.compensation_mean)))

  def states():
    return np.stack([np.concatenate([np.asarray(raw(v), f32).reshape(-1) for v in vs]) for _, vs in tasks])

  for step in range(STEPS):
    ids = TASK_IDS[step]
    scale = np.asarray(REWARD_SCALE, f32)[ids]
    ll = rng.normal(size=(T1, B, A)).astype(f32); bl = rng.normal(size=(T1, B, A)).astype(f32)
    lb = (rng.normal(size=(T1, B)) * 3).astype(f32); act = rng.integers(0, A, (T1, B))
    rew = ((rng.normal(size=(T1, B)) * 2 + 3) * scale).astype(f32); done = rng.random((T1, B)) < 0.1
    p = '%d_' % step
    out.update({p + 'll': ll, p + 'lb': lb, p + 'bl': bl, p + 'act': act, p + 'rew': rew, p + 'done': done,
                p + 'task_ids': ids, p + 'state_before': states()})
    vs_all, pg_all, adv_all, tlp_all, e_all = (np.zeros((T1 - 1, B), f32) for _ in range(5))
    for k, (pa, _) in enumerate(tasks):
      cols = np.nonzero(ids == k)[0]
      if cols.size == 0:
        continue
      a = act[:-1][:, cols]
      tlp = np.take_along_axis(_log_softmax(ll[:-1][:, cols]), a[..., None], -1)[..., 0]
      blp = np.take_along_axis(_log_softmax(bl[:-1][:, cols]), a[..., None], -1)[..., 0]
      disc = ((~done[1:][:, cols]).astype(f32) * f32(discounting)).astype(f32)
      u = pa.unnormalize_prediction(pa.correct_prediction(T(lb[:, cols])))
      ret = vtrace.from_importance_weights(T(tlp), T(blp), T(disc), T(rew[1:][:, cols]), u[:-1], u[-1],
                                           lambda_=lambda_)
      n = pa.normalize_target(ret.vs)
      adv = pa.normalize_advantage(ret.pg_advantages)
      del logged[:]
      pa.update_normalization_statistics(ret.vs)
      e = raw(n) - raw(pa.correct_prediction(T(lb[:-1][:, cols])))
      vs_all[:, cols] = raw(ret.vs)
      pg_all[:, cols] = raw(ret.pg_advantages)
      adv_all[:, cols] = raw(adv)
      tlp_all[:, cols] = tlp
      e_all[:, cols] = e
    # the loss terms of the whole batch: every mean over all (T1-1) x B rows
    out.update({p + 'vs': vs_all, p + 'pg_adv': pg_all, p + 'adv': adv_all, p + 'e': e_all,
                p + 'state_after': states(), p + 'policy_loss': -np.mean(tlp_all * adv_all, dtype=f32),
                p + 'v_loss': f32(baseline_cost) * f32(0.5) * np.mean(e_all * e_all, dtype=f32)})
  np.savez_compressed(os.path.join(HERE, 'popart_tasks_golden.npz'), **out)
  print('wrote popart_tasks_golden.npz:', len(out), 'arrays')


if __name__ == '__main__':
  main()
