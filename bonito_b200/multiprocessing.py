"""
`thread_iter`: run an iterator on a background thread with a bounded queue, the only piece of
`bonito/multiprocessing.py` (lines 20-24, 92-122) on the chunked GPU path.
"""

import queue
from threading import Thread

_DONE = object()


class ThreadIterator(Thread):
    def __init__(self, iterator, maxsize=1):
        super().__init__(daemon=True)
        self.iterator = iterator
        self.queue = queue.Queue(maxsize)
        self.error = None

    def run(self):
        try:
            for item in self.iterator:
                self.queue.put(item)
        except BaseException as err:  # surface producer failures on the consumer thread
            self.error = err
        self.queue.put(_DONE)

    def __iter__(self):
        self.start()
        while True:
            item = self.queue.get()
            if item is _DONE:
                break
            yield item
        if self.error is not None:
            raise self.error


def thread_iter(iterator, maxsize=1):
    return iter(ThreadIterator(iterator, maxsize=maxsize))
