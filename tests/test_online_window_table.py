"""The window table the density training kernels sample the online stream from (``data.sampler.window_table``),
decoded by a transcription of the kernels' ``stream_row``: every draw equals the one ``OnlineWindowSchedule`` makes."""
import numpy as np
import pytest

from nn_distributed_training_b200.data.sampler import WIN_MAX, OnlineWindowSchedule, window_table

from window_oracle import CASES, schedule_rows, stream_rows

SEED = 5


@pytest.mark.parametrize("case", sorted(CASES))
def test_window_table_decodes_to_schedule_draws(case):
    geoms, B, launches = CASES[case]
    scheds = [OnlineWindowSchedule(*g) for g in geoms]
    tab = window_table(scheds)
    assert tab.shape == (len(geoms), 2 + (WIN_MAX + 1) + 2 * WIN_MAX)
    for node0 in (0, 7):
        for calls in launches:
            for l, ((T, S, _), sch) in enumerate(zip(geoms, scheds)):
                m = T * S
                got = stream_rows(tab[l], m, B, calls[l], SEED, node0 + l)
                want = schedule_rows(sch, m, B, calls[l], SEED, node0 + l)
                np.testing.assert_array_equal(got, want, err_msg=f"{case} node {l} call {calls[l]} node0 {node0}")
                assert got.min() >= 0 and got.max() < m


def test_window_table_layout():
    """Period, window count and bounds of the geometries the kernels rely on: P != m when the last scan is never
    drawn, exactly kWinMax windows, and the paper trajectory's short last window."""
    tab = window_table([OnlineWindowSchedule(10, 7, 3), OnlineWindowSchedule(129, 3, 2),
                        OnlineWindowSchedule(2430, 500, 800)])
    K = WIN_MAX
    assert (tab[0, 0], tab[0, 1]) == (3, 63)
    assert list(tab[0, 2: 6]) == [0, 21, 42, 63]
    assert list(tab[0, 2 + K + 1: 2 + K + 4]) == [0, 21, 42] and list(tab[0, 2 + 2 * K + 1: 2 + 2 * K + 4]) == [21, 42, 63]
    assert (tab[1, 0], tab[1, 1]) == (64, 384)
    assert (tab[2, 0], tab[2, 1]) == (4, 2430 * 500)
    assert (tab[2, 2 + K + 4], tab[2, 2 + 2 * K + 4]) == (1200000, 1215000)
    assert not tab[0, 2 + 4: 2 + K + 1].any() and not tab[0, 2 + K + 4: 2 + 2 * K + 1].any()


def test_window_table_refuses_more_than_64_windows():
    window_table([OnlineWindowSchedule(129, 3, 2)])
    with pytest.raises(RuntimeError, match="more than 64 windows"):
        window_table([OnlineWindowSchedule(130, 3, 2)])
