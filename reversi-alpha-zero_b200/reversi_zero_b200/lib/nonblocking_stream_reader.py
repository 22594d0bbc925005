"""Line reader over a blocking stream (reference lib/nonblocking_stream_reader.py): a daemon thread reads lines into a
queue, so the NBoard engine's main loop can poll stdin with a timeout while a search runs, and a callback sees every
line the moment it arrives (``ping`` interrupts a search that way)."""
from logging import getLogger
from queue import Queue, Empty
from threading import Thread

logger = getLogger(__name__)


class NonBlockingStreamReader:
    def __init__(self, stream):
        self._stream = stream
        self._queue = Queue()
        self._thread = None
        self.closed = True

    def start(self, push_callback=None):
        def _worker():
            while True:
                line = self._stream.readline()
                if line:
                    if push_callback:
                        push_callback(line)
                    self._queue.put(line)
                else:
                    logger.debug("the stream may be closed")
                    break
            self.closed = True

        self._thread = Thread(target=_worker, name=f"NonBlockingStreamReader of {self._stream!r}", daemon=True)
        self.closed = False
        self._thread.start()

    def readline(self, timeout=None):
        try:
            return self._queue.get(block=timeout is not None, timeout=timeout)
        except Empty:
            return None
