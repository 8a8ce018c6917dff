"""IMPALA training script in the shape of the reference's examples/IMPALA/train.py (Learner with sampling threads, a
bounded sample queue, a learn thread, stale parameter broadcast, schedulers, WindowStat / TimeStat metrics) running on
parl_b200: the remote Actor is the DEVICE actor pool (one actor = thousands of lock-stepped envs on the GPU) and the
agent's learn() is the wgmma learner.  Only the imports differ from a reference-style script:

    import parl_b200; parl_b200.install_as_parl()      # then: import parl ... exactly as with PaddlePaddle/PARL

    python examples/impala_train.py --seconds 20 --env_num 1024
"""
import argparse
import os
import queue
import sys
import threading
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import parl_b200  # noqa: E402

parl_b200.install_as_parl()
import parl  # noqa: E402
from parl.utils import logger  # noqa: E402
from parl.utils.scheduler import PiecewiseScheduler  # noqa: E402
from parl.utils.time_stat import TimeStat  # noqa: E402
from parl.utils.window_stat import WindowStat  # noqa: E402
from parl_b200.engine.impala_host import DeviceImpalaActor, AtariAgent  # noqa: E402

config = {
    'master_address': 'localhost:8010',
    'actor_num': 1,                      # one device pool per GPU replaces the reference's 32 CPU actors x 5 envs
    'env_num': 1024,
    'sample_batch_steps': 50,
    'sample_queue_max_size': 2,
    'gamma': 0.99,
    'vf_loss_coeff': 0.5,
    'clip_rho_threshold': 1.0,
    'clip_pg_rho_threshold': 1.0,
    'lr_scheduler': [(0, 0.001), (20000, 0.0005), (40000, 0.0001)],
    'entropy_coeff_scheduler': [(0, -0.01)],
    'get_remote_metrics_interval': 10,
    'log_metrics_interval_s': 5,
    'params_broadcast_interval': 1,
}

Actor = parl.remote_class(wait=False)(DeviceImpalaActor)


class Learner(object):
    def __init__(self, cfg):
        self.config = cfg
        self.sample_data_queue = queue.Queue(maxsize=cfg['sample_queue_max_size'])
        self.agent = AtariAgent(cfg)
        self.cache_params = self.agent.get_weights()
        self.params_lock = threading.Lock()
        self.params_updated = False
        self.cache_params_sent_cnt = 0
        self.lr_scheduler = PiecewiseScheduler(cfg['lr_scheduler'])
        self.entropy_coeff_scheduler = PiecewiseScheduler(cfg['entropy_coeff_scheduler'])
        self.total_loss_stat, self.kl_stat = WindowStat(100), WindowStat(100)
        self.learn_time_stat = TimeStat(100)
        self.sample_total_steps = 0
        self.remote_metrics_queue = queue.Queue()
        self.stop = False
        self.start_time = time.time()
        self.learn_thread = threading.Thread(target=self.run_learn, daemon=True)
        self.learn_thread.start()
        parl.connect(cfg['master_address'])
        self.sample_threads = [threading.Thread(target=self.run_remote_sample, daemon=True)
                               for _ in range(cfg['actor_num'])]
        for t in self.sample_threads:
            t.start()

    def run_learn(self):
        while not self.stop:
            try:
                batch = self.sample_data_queue.get(timeout=0.2)
            except queue.Empty:
                continue
            self.sample_total_steps += batch['obs'].shape[0]
            lr, ent = self.lr_scheduler.step(1), self.entropy_coeff_scheduler.step(1)
            with self.learn_time_stat:
                total_loss, pi_loss, vf_loss, entropy, kl = self.agent.learn(
                    batch['obs'], batch['actions'], batch['behaviour_logits'], batch['rewards'], batch['dones'], lr, ent)
            self.params_updated = True
            self.total_loss_stat.add(total_loss)
            self.kl_stat.add(kl)

    def run_remote_sample(self):
        remote_actor = Actor(self.config)
        cnt = 0
        remote_actor.set_weights(self.cache_params).get()
        while not self.stop:
            batch = remote_actor.sample().get()
            while not self.stop:
                try:
                    self.sample_data_queue.put(batch, timeout=0.2)
                    break
                except queue.Full:
                    continue
            cnt += 1
            if cnt % self.config['get_remote_metrics_interval'] == 0:
                metrics = remote_actor.get_metrics().get()
                if metrics['episode_rewards']:
                    self.remote_metrics_queue.put(metrics)
            with self.params_lock:
                if self.params_updated and self.cache_params_sent_cnt >= self.config['params_broadcast_interval']:
                    self.params_updated = False
                    self.cache_params = self.agent.get_weights()
                    self.cache_params_sent_cnt = 0
                self.cache_params_sent_cnt += 1
            remote_actor.set_weights(self.cache_params).get()
        remote_actor.destroy()

    def log_metrics(self):
        rewards = []
        while True:
            try:
                rewards.extend(self.remote_metrics_queue.get_nowait()['episode_rewards'])
            except queue.Empty:
                break
        el = time.time() - self.start_time
        logger.info({'sample_steps': self.sample_total_steps, 'env_steps_per_s': int(self.sample_total_steps / max(el, 1e-9)),
                     'mean_episode_rewards': (sum(rewards) / len(rewards)) if rewards else None,
                     'total_loss': self.total_loss_stat.mean, 'kl': self.kl_stat.mean,
                     'learn_time_s': self.learn_time_stat.mean, 'elapsed_time_s': int(el)})


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--seconds', type=float, default=20.0)
    ap.add_argument('--env_num', type=int, default=config['env_num'])
    args = ap.parse_args()
    config['env_num'] = args.env_num
    learner = Learner(config)
    t_end = time.time() + args.seconds
    while time.time() < t_end:
        time.sleep(config['log_metrics_interval_s'])
        learner.log_metrics()
    learner.stop = True
    time.sleep(1.0)
    learner.log_metrics()
