"""CPU: the host handshake of StyleTransfer(devices=[a, b]) (style_transfer._Lockstep) on two plain threads.

Each rank runs the hook sequence of StyleTransfer._stylize's iteration loop around a fake launch; rank 0's callback
makes the collective gathers get_image() makes on a banded scale.  What must hold: both ranks launch the same steps
however either one stops, and every gather rank 0 requests pairs with rank 1's rows of the very step rank 0 reports.
"""
import random
import signal
import threading
import time

import pytest

from style_transfer_b200.style_transfer import _Lockstep, _Stopped, _deferred_sigint


class _Rank:
    def __init__(self, rank, sync, bar, fail_serving=None):
        self._rank, self.sync, self.bar = rank, sync, bar
        self.launched, self.gathered = [], []
        self.fail_serving = fail_serving

    def get_image_tensor(self):
        if self._rank == 0:
            self.sync.request_gather()
        self.gathered.append(self.launched[-1])
        self.bar.wait()
        if self.fail_serving == self.launched[-1]:    # fails after the collective part: rank 0's gather succeeded
            raise RuntimeError('rank 1 failed while serving')


def _loop(st, scales, callback, fail_before_launch=None, sigint_in_launch=None):
    sync, step = st.sync, 0
    for its in scales:
        for _ in range(its):
            if fail_before_launch == step + 1:
                raise RuntimeError('rank 1 failed')
            sync.before_launch(st, step + 1)
            time.sleep(random.random() * 1e-3)
            step += 1
            st.launched.append(step)
            if sigint_in_launch == step:        # Ctrl-C while the launch call runs: lands right after it returns
                signal.raise_signal(signal.SIGINT)
            sync.after_launch(st, step)
            if callback is not None:
                callback(st, step)
            sync.after_iteration(st, step)
        sync.end_of_scale(st, step)


def _drive(scales, cb0=None, fail1=None, fail_serving=None, sigint0=None):
    """Rank 0 on this (the main) thread under _deferred_sigint, as StyleTransfer._stylize_devices runs it."""
    sync, bar = _Lockstep(), threading.Barrier(2)
    ranks = [_Rank(0, sync, bar), _Rank(1, sync, bar, fail_serving)]
    errors = [None, None]

    def run(r):
        try:
            _loop(ranks[r], scales, cb0 if r == 0 else None, fail1 if r == 1 else None, sigint0 if r == 0 else None)
        except BaseException as e:  # noqa: BLE001
            errors[r] = e
            sync.stop()
            bar.abort()

    t = threading.Thread(target=run, args=(1,))
    with _deferred_sigint(sync):
        t.start()
        run(0)
        t.join(30)
    assert not t.is_alive()
    return ranks, errors


@pytest.mark.parametrize('seed', range(4))
def test_gathers_pair_with_the_reported_step(seed):
    random.seed(seed)

    def cb(st, step):
        for _ in range(step % 3):     # zero, one or two get_image() calls per iteration
            st.get_image_tensor()

    ranks, errors = _drive([5, 4, 6], cb)
    assert errors == [None, None]
    assert ranks[0].launched == ranks[1].launched == list(range(1, 16))
    assert ranks[1].gathered == ranks[0].gathered
    assert len(ranks[0].gathered) == sum(s % 3 for s in range(1, 16))


@pytest.mark.parametrize('seed', range(4))
def test_callback_error_leaves_equal_launches(seed):
    random.seed(seed)

    def cb(st, step):
        st.get_image_tensor()
        if step == 3:
            raise ValueError('callback')

    ranks, errors = _drive([6], cb)
    assert isinstance(errors[0], ValueError) and isinstance(errors[1], _Stopped)
    assert ranks[0].launched == ranks[1].launched == [1, 2, 3]


def test_rank1_error_stops_rank0_before_its_launch():
    ranks, errors = _drive([6], fail1=4)
    assert isinstance(errors[1], RuntimeError) and isinstance(errors[0], _Stopped)
    assert ranks[0].launched == ranks[1].launched == [1, 2, 3]


@pytest.mark.parametrize('seed', range(4))
def test_ctrl_c_during_a_launch_stops_at_the_next_gate(seed):
    """SIGINT that lands between rank 0's launch and its publication is held back: KeyboardInterrupt comes at rank 0's
    next gate, after rank 1 has launched the partner of that launch."""
    random.seed(seed)
    assert threading.current_thread() is threading.main_thread()
    ranks, errors = _drive([6], sigint0=3)
    assert isinstance(errors[0], KeyboardInterrupt) and isinstance(errors[1], _Stopped)
    assert ranks[0].launched == ranks[1].launched == [1, 2, 3]
    assert signal.getsignal(signal.SIGINT) is signal.default_int_handler


@pytest.mark.parametrize('seed', range(4))
def test_rank1_error_while_serving_a_gather_stops_rank0(seed):
    """Rank 1 fails serving a gather of step 2 once both passed its barrier: rank 1 never announced step 3, so rank 0
    stops at its gate instead of launching 3 alone (or, when the abort overtakes its wake-up, in that barrier)."""
    random.seed(seed)
    ranks, errors = _drive([6], cb0=lambda st, step: st.get_image_tensor(), fail_serving=2)
    assert isinstance(errors[1], RuntimeError)
    assert isinstance(errors[0], (_Stopped, threading.BrokenBarrierError))
    assert ranks[0].launched == ranks[1].launched == [1, 2]
