"""``parl.utils.summary`` surface (parl/utils/summary.py:15-18, tensorboard.py:25-46): add_scalar /
add_histogram / flush, lazily bound to tensorboardX when installed, otherwise a CSV file in the
logger directory (tensorboardX is absent from the H100 image)."""
import os

from .logger import logger

_writer = None
_csv = None


def _get():
    global _writer, _csv
    if _writer is None and _csv is None:
        logdir = logger.get_dir()
        if logdir is None:
            logger.auto_set_dir()
            logdir = logger.get_dir()
        try:
            from tensorboardX import SummaryWriter
            _writer = SummaryWriter(logdir=logdir)
        except Exception:
            _csv = open(os.path.join(logdir, 'summary.csv'), 'a')
    return _writer, _csv


def add_scalar(tag, scalar_value, global_step=None):
    w, c = _get()
    if w is not None:
        w.add_scalar(tag, scalar_value, global_step)
    else:
        c.write('%s,%s,%s\n' % (tag, global_step, float(scalar_value)))


def add_histogram(tag, values, global_step=None):
    w, _ = _get()
    if w is not None:
        w.add_histogram(tag, values, global_step)


def flush():
    w, c = _get()
    if w is not None:
        w.flush()
    else:
        c.flush()
