"""Log-line formats.  The worker line is a de-facto API: the LR-tuning parser
greps/regex-parses it (``/root/reference/src/tiny_tuning_parser.py:13-27``,
format at ``distributed_worker.py:255-258``); the PS line is
``sync_replicas_master_nn.py:221``."""

WORKER_FMT = ("Worker: {}, Step: {}, Epoch: {} [{}/{} ({:.0f}%)], Loss: {:.4f}, Time Cost: {:.4f}, "
              "Comp: {:.4f}, Encode: {: .4f}, Comm: {: .4f}, Msg(MB): {: .4f}, Prec@1: {: .4f}, Prec@5: {: .4f}")
MASTER_FMT = "Master: Step: {}, Decode Cost: {}, Cur lr {}, Gather: {}"
TEST_FMT = "Test set: Step: {}, Average loss: {:.4f}, Prec@1: {} Prec@5: {}"
EMA_TEST_FMT = "Test set (EMA): Step: {}, Average loss: {:.4f}, Prec@1: {} Prec@5: {}"   # the weight average


def worker_line(rank, step, epoch, seen, total, loss, time_cost, comp, encode, comm, msg_mb, prec1, prec5):
    pct = 100.0 * seen / max(total, 1)
    return WORKER_FMT.format(rank, step, epoch, seen, total, pct, loss, time_cost, comp, encode, comm,
                             msg_mb, prec1, prec5)


def master_line(step, decode_cost, lr, gather):
    return MASTER_FMT.format(step, decode_cost, lr, gather)


def test_line(step, loss, prec1, prec5):
    return TEST_FMT.format(step, loss, prec1, prec5)


def ema_test_line(step, loss, prec1, prec5):
    return EMA_TEST_FMT.format(step, loss, prec1, prec5)


class MetricsWriter:
    """Machine-readable twin of the log lines (the reference has print() only, SURVEY 5.5): one JSON object per
    line in ``<path>.rank<R>.jsonl`` — worker records carry the worker-line fields, PS records the PS-line fields plus
    the aggregation bookkeeping.  ``path`` empty = disabled (every method is a no-op)."""

    def __init__(self, path: str, rank: int, role: str):
        import json
        import time
        self._json, self._time = json, time
        self.rank, self.role = rank, role
        self._f = open("%s.rank%d.jsonl" % (path, rank), "a") if path else None

    def write(self, **fields):
        if self._f is None:
            return
        rec = {"t": round(self._time.time(), 3), "role": self.role, "rank": self.rank}
        rec.update({k: (float(v) if isinstance(v, float) else v) for k, v in fields.items()})
        self._f.write(self._json.dumps(rec) + "\n")
        self._f.flush()

    def close(self):
        if self._f is not None:
            self._f.close()
            self._f = None
