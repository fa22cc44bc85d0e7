"""ParamLayout's padded hidden size on the CPU: every rnn_units in [1, 1024] gets the smallest Hp the session-cell
recurrence kernels run (32, 64, ..., 1024), sizes outside that range are refused when the layout is built, and the
logical <-> internal mapping stays exact with zero padding at hidden sizes that are not a kernel size themselves."""
import numpy as np
import pytest

from chameleon_recsys_b200.harness import make_problem
from chameleon_recsys_b200.plan import HP_SIZES, ParamLayout


@pytest.mark.parametrize('H, Hp', [(1, 32), (16, 32), (30, 32), (32, 32), (33, 64), (64, 64), (100, 128), (255, 256),
                                   (256, 256), (300, 512), (512, 512), (513, 1024), (1024, 1024)])
def test_hidden_size_pads_to_a_recurrence_kernel_size(H, Hp):
    pb = make_problem('tiny', profile='B', rnn_units=H)
    assert pb.layout.Hp == Hp
    assert Hp in HP_SIZES


@pytest.mark.parametrize('H', [0, -1, 1025, 2048])
def test_hidden_size_outside_the_kernel_range_is_refused(H):
    pb = make_problem('tiny', profile='B')
    with pytest.raises(ValueError, match='rnn_units'):
        ParamLayout(pb.plan, pb.hp.CAR_embedding_size, H, 1)


@pytest.mark.parametrize('cell', ['ugrnn', 'gru', 'lstm'])
@pytest.mark.parametrize('H', [100, 300])
def test_round_trip_and_zero_padding(cell, H):
    """Two layers: logical -> internal -> logical is exact, every recurrent and W3 block is Hp rows (and Hp-wide column
    blocks), and nothing lands outside the logical entries' slots."""
    pb = make_problem('tiny', profile='B', rnn_cell=cell, rnn_units=H, rnn_num_layers=2)
    lay = pb.layout
    Hp = lay.Hp
    G = {'ugrnn': 2, 'gru': 3, 'lstm': 4}[cell]
    rs = np.random.RandomState(H)
    lg = {k: (rs.rand(*v.shape) + 0.5).astype(np.float32) for k, v in lay.init_logical(1).items()}   # no zeros
    flat = lay.to_internal(lg)
    back = lay.to_logical(flat)
    assert sorted(back) == sorted(lg)
    for k in lg:
        assert np.array_equal(back[k], lg[k]), (cell, H, k)
    # every logical entry has its own slot: the nonzeros of the flat buffer are exactly the logical entries
    assert np.count_nonzero(flat) == sum(v.size for v in lg.values())
    assert lay.by_key['W3'].rows == Hp
    for i in range(2):
        assert lay.by_key['rnn%d/Wx' % i].rows == (lay.C if i == 0 else Hp)
        assert lay.by_key['rnn%d/Wx' % i].ld == G * Hp
        assert lay.by_key['rnn%d/Wh' % i].rows == Hp
        wx = flat[lay.by_key['rnn%d/Wx' % i].offset:][:lay.by_key['rnn%d/Wx' % i].size].reshape(-1, G * Hp)
        for g in range(G):
            assert not wx[:, g * Hp + H:(g + 1) * Hp].any()
        if i == 1:
            assert not wx[H:].any()
