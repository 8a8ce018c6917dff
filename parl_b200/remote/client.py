"""``parl.connect`` façade (parl/remote/client.py:405-448).

In the reference, connect() attaches the process to an xparl master that hands out CPU jobs.
Here the "cluster" is the local H100(s): connect() records the address (kept only for logging /
API compatibility), probes the visible devices and enables instantiation of ``@remote_class``
objects, which are hosted in-process on the device actor pool — no ZeroMQ, no cloudpickle, no
subprocesses.  Instantiating a remote class before connect() raises the reference's assertion."""
import threading

_client = None
_lock = threading.Lock()


class Client(object):
    def __init__(self, master_address, distributed_files=()):
        import torch
        self.master_address = master_address
        self.distributed_files = list(distributed_files or [])
        self.n_devices = torch.cuda.device_count() if torch.cuda.is_available() else 0
        self.actor_num = 0
        self._next_device = 0
        self.lock = threading.Lock()

    def allocate_device(self, n_gpu=0):
        """Round-robin placement hint for hosted objects (n_gpu mirrors remote_class(n_gpu=...))."""
        with self.lock:
            self.actor_num += 1
            if self.n_devices == 0:
                return None
            d = self._next_device
            self._next_device = (self._next_device + 1) % self.n_devices
            return d


def connect(master_address, distributed_files=[]):
    """Same signature as the reference; ``distributed_files`` are not shipped anywhere because
    remote objects live in this process."""
    global _client
    assert isinstance(master_address, str) and len(master_address) > 0
    with _lock:
        _client = Client(master_address, distributed_files)
    return _client


def get_global_client():
    assert _client is not None, "Cannot instantiate a remote class before calling parl.connect() " \
                                "(please call `parl.connect(master_address)` first)."
    return _client


def disconnect():
    global _client
    with _lock:
        _client = None
