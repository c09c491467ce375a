"""engine.pipelined, the two-in-flight loop behind forward_batches, the inference driver and evaluate_rows, driven by
fake submit / wait / retire callables that record their calls: submission i + 1 precedes the wait for i, and every
submission not waited for is retired exactly once when a submit or a wait raises or the consumer stops early."""
import pytest

from deepconsensus_b200 import engine


class Fake:
  def __init__(self, fail_submit=None, fail_wait=None):
    self.calls, self.fail_submit, self.fail_wait = [], fail_submit, fail_wait

  def submit(self, item):
    self.calls.append(("submit", item))
    if item == self.fail_submit:
      raise engine.DcbError(-1, "submit %s" % item)
    return "h%s" % item

  def wait(self, handle):
    self.calls.append(("wait", handle))
    if handle == "h%s" % self.fail_wait:
      raise engine.DcbError(-5, "wait %s" % handle)
    return handle.upper()

  def retire(self, handle):
    self.calls.append(("retire", handle))

  def run(self, items):
    return engine.pipelined(items, self.submit, self.wait, self.retire)

  def retired(self):
    return [h for op, h in self.calls if op == "retire"]


def test_submit_wait_interleaving():
  f = Fake()
  assert list(f.run(range(3))) == [(0, "H0"), (1, "H1"), (2, "H2")]
  assert f.calls == [("submit", 0), ("submit", 1), ("wait", "h0"), ("submit", 2), ("wait", "h1"), ("wait", "h2")]
  one, none = Fake(), Fake()
  assert list(one.run([7])) == [(7, "H7")] and one.calls == [("submit", 7), ("wait", "h7")]
  assert list(none.run([])) == [] and none.calls == []


def test_failed_wait_retires_the_younger_submission():
  f = Fake(fail_wait=1)
  got = []
  with pytest.raises(engine.DcbError) as ei:
    for r in f.run(range(4)):
      got.append(r)
  assert ei.value.code == -5 and got == [(0, "H0")]
  assert f.calls[-3:] == [("submit", 2), ("wait", "h1"), ("retire", "h2")]
  assert f.retired() == ["h2"]
  last = Fake(fail_wait=2)                     # the last wait: nothing younger is in flight
  with pytest.raises(engine.DcbError):
    list(last.run(range(3)))
  assert last.retired() == []


def test_failed_submit_retires_the_older_submission():
  f = Fake(fail_submit=2)
  with pytest.raises(engine.DcbError) as ei:
    list(f.run(range(4)))
  assert ei.value.code == -1
  assert f.calls[-2:] == [("submit", 2), ("retire", "h1")]
  assert f.retired() == ["h1"]
  first = Fake(fail_submit=0)
  with pytest.raises(engine.DcbError):
    list(first.run(range(2)))
  assert first.retired() == []


def test_consumer_closing_early_retires_what_is_in_flight():
  f = Fake()
  gen = f.run(range(5))
  assert next(gen) == (0, "H0")
  gen.close()
  assert f.calls == [("submit", 0), ("submit", 1), ("wait", "h0"), ("retire", "h1")]
  raising = Fake()                             # a consumer that raises while handling a result
  with pytest.raises(KeyError):
    for item, _ in raising.run(range(5)):
      if item == 2:
        raise KeyError(item)
  assert raising.retired() == ["h3"]


def test_nothing_is_retired_twice_or_after_being_waited_for():
  cases = [Fake(fail_wait=k) for k in range(4)] + [Fake(fail_submit=k) for k in range(4)] + [Fake()]
  for f in cases:
    try:
      list(f.run(range(4)))
    except engine.DcbError:
      pass
    waited, retired = [h for op, h in f.calls if op == "wait"], f.retired()
    submitted = ["h%s" % i for op, i in f.calls if op == "submit" and i != f.fail_submit]
    assert len(set(retired)) == len(retired) and not set(retired) & set(waited)
    assert sorted(waited + retired) == sorted(submitted)           # every submission is waited for or retired
