"""Host-to-device staging shared by the front ends and the serving pipeline: RowStager copies host row arrays into
device rows, Upload keeps a small device table in step with a host value."""
import numpy as np
import torch


class RowStager:
    """H2D copies of host row arrays into device rows.  Pinned tensors are copied directly; anything else goes through
    a pinned staging buffer shaped like the device rows, allocated on first need.  The staging buffer may still feed
    the previous put's copies when the next put rewrites it, so each put waits for those first (its own event)."""

    def __init__(self):
        self.staging = None
        self.copied = None

    def put(self, arrays, dst):
        """Enqueues the H2D copies of `arrays` (float32 [n_i, dst.shape[1]] host arrays or tensors) back to back into
        the device rows dst[0:sum(n_i)]; every put of one stager has dst of the same shape.  Returns sum(n_i)."""
        at, staged = 0, False
        with torch.cuda.device(dst.device):
            for a in arrays:
                k = int(a.shape[0])
                if not k:
                    continue
                src = a
                if not (torch.is_tensor(a) and a.is_pinned()):
                    if self.staging is None:
                        self.staging = torch.empty(dst.shape, dtype=torch.float32, pin_memory=True)
                        self.copied = torch.cuda.Event()
                    if not staged:
                        self.copied.synchronize()
                        staged = True
                    src = self.staging[at:at + k]
                    src.copy_(torch.as_tensor(a))
                dst[at:at + k].copy_(src, non_blocking=True)
                at += k
            if staged:
                self.copied.record()
        return at


class Upload:
    """A small device table `dev` that goes H2D only when its bytes change, through a pinned staging copy."""

    def __init__(self, dev):
        self.dev = dev
        self.staging = torch.empty(dev.shape, dtype=dev.dtype, pin_memory=True)
        self.copied = torch.cuda.Event()
        self.last = None

    def put(self, value, always=False):
        """Enqueues the H2D copy of the host `value` (dev's shape, converted to its dtype) unless its bytes equal the
        last put's; always=True copies in any case.  Returns whether it copied."""
        host = self.staging.numpy()
        value = np.asarray(value, host.dtype)
        raw = value.tobytes()
        if raw == self.last and not always:
            return False
        self.copied.synchronize()                 # the staging buffer may still feed the previous copy
        host[...] = value
        with torch.cuda.device(self.dev.device):
            self.dev.copy_(self.staging, non_blocking=True)
            self.copied.record()
        self.last = raw
        return True
