"""The producer behind a started ``Queue`` (ae_factory.Queue.start): the reference's FIFOQueue with NUM_THREADS feeder threads
(auto_pose/ae/queue.py:14-74) as one host thread and a ring of device slots.

The thread makes each batch's random draws in ``Dataset.batch_device``'s order, uploads them and launches the indexed input
kernels on a non-blocking stream of its own, into one of ``queue_size`` slots, and records the slot's ``ready`` event.  A
``pull`` (one per ``Session.run``) makes the caller's current stream wait for that event -- the host never waits for the
device -- and hands out the slot's x / y.  The slot goes back to the producer at the next ``pull`` (or at ``close``) with an
event recorded on the consumer's stream behind the run that read it, and the producer's stream waits for that event before it
writes the slot again.  The first fill waits the same way for an event recorded when the slots were allocated, since their
memory comes from the consumer stream's pool and may still be read by work queued there.  So batches come out in draw order, with the bits of repeated synchronous calls, while the producer
runs up to ``queue_size`` batches ahead of the device.

One thread is enough (the draws and packing of a batch of 64 take well under a training step) and it is what keeps the batch
stream a function of the seeds alone: NUM_THREADS is accepted and does not change it.  The thread is the only user of numpy's
global random stream while it runs; nothing else in the package draws from it."""
import atexit
import queue
import threading
import weakref

import torch

from .. import _lib

_LIVE = weakref.WeakSet()


@atexit.register
def _close_all():
    for p in list(_LIVE):
        p.close()


class BatchProducer(object):
    def __init__(self, dataset, batch_size, queue_size, device):
        if queue_size < 1:
            raise ValueError("QUEUE_SIZE must be >= 1, got %d" % queue_size)
        self._ds = dataset
        self._batch_size = int(batch_size)
        self._device = device
        try:
            self._stacks = dataset.resident(device)
        except RuntimeError:
            dataset.upload(device)                    # the training set goes up once; later starts reuse it
            self._stacks = dataset.resident(device)
        shape = (self._batch_size,) + tuple(dataset.shape)
        with torch.cuda.device(device):
            self._stream = torch.cuda.Stream(device)        # non-blocking: not ordered against the legacy default stream
            self._slots = [(torch.empty(shape, dtype=torch.float32, device=device),
                            torch.empty(shape, dtype=torch.float32, device=device), torch.cuda.Event()) for _ in range(queue_size)]
            self._scratch = [dataset._resident_scratch(self._batch_size, device) for _ in range(queue_size)]
            # Slots and their scratch come from the caller's stream's pool: a block may have been freed there while work queued on
            # that stream still reads it.  The first fill of every slot waits for this event, so it lands behind that work.
            allocated = torch.cuda.Event()
            allocated.record(torch.cuda.current_stream(device))
        self._released = [allocated] * queue_size     # consumer-stream event after the last use of the slot's memory
        self._free = queue.Queue()
        self._filled = queue.Queue()
        for s in range(queue_size):
            self._free.put(s)
        self._held = None
        self._error = None
        self._stop = threading.Event()
        self._thread = threading.Thread(target=self._run, name="aae-batch-producer", daemon=True)
        self._thread.start()
        _LIVE.add(self)

    def _run(self):
        try:
            with torch.cuda.device(self._device), torch.cuda.stream(self._stream):
                while True:
                    s = self._free.get()
                    if s is None or self._stop.is_set():
                        return
                    draws = self._ds._draws(self._batch_size)
                    self._stream.wait_event(self._released[s])
                    x, y, ready = self._slots[s]
                    self._ds._enqueue_resident(self._stacks, draws, x, y, self._stream, scratch=self._scratch[s])
                    ready.record(self._stream)
                    self._filled.put(s)
        except BaseException as e:          # handed to the consumer: pull raises it
            self._filled.put(e)

    def _release_held(self):
        if self._held is not None:
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(self._device))
            self._released[self._held] = ev
            self._free.put(self._held)
            self._held = None

    def pull(self):
        """(x, y) float32 device tensors of the next batch, ordered on the caller's current stream.  They stay valid until the
        next pull or ``close``."""
        if self._thread is None:
            raise _lib.AaeError("the batch producer is closed")
        self._release_held()
        item = self._error if self._error is not None else self._filled.get()
        if isinstance(item, BaseException):
            self._error = item
            raise _lib.AaeError("the batch producer failed: %s" % item) from item
        x, y, ready = self._slots[item]
        torch.cuda.current_stream(self._device).wait_event(ready)
        self._held = item
        return x, y

    def close(self):
        """Stops and joins the thread; batches made ahead and not pulled are dropped.  Waits for the device, so the slots can
        be freed."""
        if self._thread is None:
            return
        self._stop.set()
        self._free.put(None)
        self._thread.join()
        self._thread = None
        self._held = None
        torch.cuda.synchronize(self._device)
        self._slots, self._scratch = [], []
        _LIVE.discard(self)
