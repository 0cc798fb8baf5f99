"""`Episode` (the record Agent.evaluate returns, base/core/utils.py:12-36), the host version of the action-smoothness
metric (:82-120; the device version is K6, csrc/smoothness.cu) and the wandb-config loader (:123-146)."""
from dataclasses import dataclass
from pathlib import Path
from typing import List

import numpy as np


@dataclass
class Episode:
    fitness: np.float64
    smoothness: np.float64
    length: np.float64
    state_history: List
    ref_signals: List
    actions: List
    reward_lst: List

    def get_history(self) -> np.ndarray:
        """Time traces [3 references | 3 actuator commands | 12 states | reward], one row per step."""
        steps = len(self.state_history)
        t_axis = np.linspace(0, self.length, steps)
        refs = np.stack([[signal(t) for t in t_axis] for signal in self.ref_signals], axis=1)
        rewards = np.asarray(self.reward_lst, dtype=np.float64).reshape(steps, 1)
        return np.hstack([refs, np.asarray(self.actions), np.asarray(self.state_history), rewards])


def calc_smoothness(y: np.ndarray, dt: float = 0.01, **kwargs) -> float:
    """-sqrt(sum over channels and frequencies of f * S_yy(f) * 2/N) * 100 * 80/T with S_yy = |FFT(y)|^2 dt over the
    bins 1 .. N/2-1 and f = linspace(dt, 1/(2 dt), N/2-1)."""
    n_samples = y.shape[0]
    bins = n_samples // 2 - 1
    if bins <= 0:
        return -0.0
    spectrum = np.fft.fft(np.asarray(y, dtype=np.float64), n_samples, axis=0)[1:n_samples // 2]
    power = np.abs(spectrum * np.conjugate(spectrum)) * dt
    freq = np.linspace(dt, 1 / (2 * dt), bins)
    roughness_per_channel = (freq[:, None] * power).sum(axis=0) * 2 / n_samples
    return -(np.sqrt(roughness_per_channel.sum()) * 100 * (80 / (n_samples * dt)))


def calc_nMAE(error: np.ndarray) -> float:
    """Normalised mean absolute tracking error in % (base/core/utils.py:39-58): per-channel mean |error| over ranges of 20 deg
    for theta and phi and max(|mean beta error|, 3.14159/180) for beta, averaged over the three channels."""
    err = np.asarray(error, dtype=np.float64)
    mae = np.abs(err).mean(axis=0)
    ranges = np.array([np.deg2rad(20), np.deg2rad(20), max(abs(err[:, -1].mean()), 3.14159 / 180)])
    return float(np.mean(mae / ranges) * 100)


def load_config(model_path: str, verbose: bool = False) -> dict:
    """Read `<run>/files/config.yaml` as written by wandb ({key: {value: v, desc: ...}}) into a flat dict."""
    import yaml
    raw = yaml.safe_load((Path(model_path) / 'files' / 'config.yaml').read_text(encoding='utf-8'))
    flat = {key: (entry['value'] if isinstance(entry, dict) else entry) for key, entry in raw.items()}
    if verbose:
        print(flat)
    return flat
