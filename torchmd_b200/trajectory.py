"""Trajectory and log output without stalling the MD loop (SURVEY.md section 8f-4).

The reference's loop (run.py:257-291) copies the positions to the host synchronously every
output period, keeps every frame in a Python list and re-saves the WHOLE trajectory with
``np.save(np.stack(frames, axis=2))`` at every save period ("ideally we want to append").
Here:

* ``NpyAppender`` writes the same file -- ``np.load`` returns the same ``(natoms, 3, nframes)``
  array -- but appendable: the array is declared Fortran-ordered, so frame ``f`` is one
  contiguous block of ``3*natoms`` values (x of all atoms, then y, then z) at the end of the
  file, and only the fixed-size header is rewritten when the frame count changes.
* ``FrameSink`` takes a snapshot of ``system.pos`` with a transposing copy on a side stream into
  one of two pinned host buffers and hands it to a writer thread: the compute stream only
  waits for an event, the host never waits for the disk (it waits only if both buffers are
  still in flight).
* ``LogWriter`` is the reference's CSV monitor (utils.py:10-38), same columns and file layout.
"""
import csv
import json
import os
import queue
import threading
import time

import numpy as np
import torch

_HEADER_BYTES = 256  # magic(6) + version(2) + header length(2) + dict padded with spaces + newline


class NpyAppender:
    """``(natoms, 3, nframes)`` .npy file that grows by whole frames."""

    def __init__(self, path, natoms, dtype=np.float32):
        self.path, self.natoms, self.dtype = path, int(natoms), np.dtype(dtype)
        self.nframes = 0
        d = os.path.dirname(path)
        if d:
            os.makedirs(d, exist_ok=True)
        self._fh = open(path, "w+b")
        self._write_header()

    def _write_header(self):
        body = "{'descr': %r, 'fortran_order': True, 'shape': (%d, 3, %d), }" % (self.dtype.str, self.natoms, self.nframes)
        room = _HEADER_BYTES - 10 - 1
        if len(body) > room:
            raise ValueError("npy header does not fit its reserved space")
        header = b"\x93NUMPY\x01\x00" + (_HEADER_BYTES - 10).to_bytes(2, "little") + body.ljust(room).encode("latin1") + b"\n"
        self._fh.seek(0)
        self._fh.write(header)

    def append(self, frame_xyz_major):
        """``frame_xyz_major``: (3, natoms) array -- x of all atoms, y, z -- of the file's dtype."""
        a = np.ascontiguousarray(frame_xyz_major, dtype=self.dtype)
        if a.shape != (3, self.natoms):
            raise ValueError(f"frame has shape {a.shape}, expected (3, {self.natoms})")
        self._fh.seek(_HEADER_BYTES + self.nframes * 3 * self.natoms * self.dtype.itemsize)
        self._fh.write(a.tobytes())
        self.nframes += 1

    def flush(self):
        """Make the file loadable up to the frames appended so far."""
        self._write_header()
        self._fh.flush()

    def close(self):
        if self._fh is not None:
            self.flush()
            self._fh.close()
            self._fh = None


class FrameSink:
    """Asynchronous trajectory output for every replica of a ``System``.

    ``snapshot(pos)`` is called where the reference does ``system.pos.detach().cpu().numpy()``
    (run.py:267): it enqueues a device-side transpose into a staging tensor and its copy into
    pinned host memory on a side stream and returns; a writer thread appends the frames to
    ``<prefix>_<replica><ext>`` once the copy has completed.  ``save_every``: rewrite the headers
    (make the files loadable) every that many snapshots, like the reference's save period.
    ``dtype``: of the staging buffers and the files -- torch.float64 for a "precision: double" run
    (the positions' dtype); the default keeps fp32 files.
    """

    def __init__(self, prefix, ext, natoms, nreplicas, device, save_every=1, nbuffers=2, dtype=torch.float32):
        self.natoms, self.nrep = int(natoms), int(nreplicas)
        self.device = torch.device(device)
        self.cuda = self.device.type == "cuda"
        if dtype not in (torch.float32, torch.float64):
            raise ValueError(f"FrameSink writes float32 or float64 frames, not {dtype}")
        self.files = [NpyAppender(f"{prefix}_{k}{ext}", natoms, dtype=np.float64 if dtype == torch.float64 else np.float32)
                      for k in range(self.nrep)]
        self.save_every = max(1, int(save_every))
        self._count = 0
        self._stage = [torch.empty((self.nrep, 3, self.natoms), dtype=dtype, device=self.device) for _ in range(nbuffers)]
        self._host = [torch.empty((self.nrep, 3, self.natoms), dtype=dtype, pin_memory=self.cuda) for _ in range(nbuffers)]
        self._free = queue.Queue()
        for b in range(nbuffers):
            self._free.put(b)
        self._work = queue.Queue()
        self._stream = torch.cuda.Stream(device=self.device) if self.cuda else None
        self._error = None
        self._thread = threading.Thread(target=self._writer, daemon=True)
        self._thread.start()

    def snapshot(self, pos):
        if self._error is not None:
            raise RuntimeError("trajectory writer failed") from self._error
        b = self._free.get()  # blocks only while every buffer is still being copied or written
        self._count += 1
        flush = self._count % self.save_every == 0
        if self.cuda:
            ready = torch.cuda.Event()
            ready.record(torch.cuda.current_stream(self.device))
            staged, done = torch.cuda.Event(), torch.cuda.Event()
            with torch.cuda.stream(self._stream):
                self._stream.wait_event(ready)
                self._stage[b].copy_(pos.detach().transpose(1, 2))  # (R,N,3) -> (R,3,N): a frame is one block of the file
                staged.record(self._stream)
                self._host[b].copy_(self._stage[b], non_blocking=True)
                done.record(self._stream)
            # the next integration step may overwrite pos: it waits for the device-side transpose only,
            # the copy to the host and the file write overlap with the following steps
            torch.cuda.current_stream(self.device).wait_event(staged)
        else:
            done = None
            self._host[b].copy_(pos.detach().transpose(1, 2))
        self._work.put((b, done, flush))

    def _writer(self):
        while True:
            item = self._work.get()
            if item is None:
                return
            b, done, flush = item
            try:
                if done is not None:
                    done.synchronize()
                frames = self._host[b].numpy()
                for k, f in enumerate(self.files):
                    f.append(frames[k])
                    if flush:
                        f.flush()
            except Exception as err:  # surfaced by the next snapshot()/close()
                self._error = err
            finally:
                self._free.put(b)
                self._work.task_done()

    def close(self):
        self._work.put(None)
        self._thread.join()
        for f in self.files:
            f.close()
        if self._error is not None:
            raise RuntimeError("trajectory writer failed") from self._error


class LogWriter:
    """utils.py:10-38: CSV monitor with the given keys plus the wall-clock column ``t``."""

    def __init__(self, path, keys, header="", name="monitor.csv"):
        self.keys = tuple(keys) + ("t",)
        assert path is not None
        os.makedirs(path, exist_ok=True)
        filename = os.path.join(path, name)
        if os.path.exists(filename):
            os.remove(filename)
        self.f = open(filename, "wt")
        if isinstance(header, dict):
            header = "# {} \n".format(json.dumps(header))
        self.f.write(header)
        self.logger = csv.DictWriter(self.f, fieldnames=self.keys)
        self.logger.writeheader()
        self.f.flush()
        self.tstart = time.time()

    def write_row(self, epinfo):
        if self.logger:
            epinfo["t"] = time.time() - self.tstart
            self.logger.writerow(epinfo)
            self.f.flush()
