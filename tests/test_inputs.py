"""BlockData / GPPPInput / split: bit-exact integer semantics.
Ports Stheno.jl test/input_collection_types.jl:4-49 and
test/gaussian_process_probabilistic_programme.jl:3-15 (+ the split doctest, gppp.jl:90-102),
for BOTH the product's host classes and the oracle's."""
import numpy as np
import pytest


@pytest.fixture(params=["product", "oracle"])
def m(request, sb, orc):
    return sb if request.param == "product" else orc


def test_blockdata(m):
    rng = np.random.default_rng(123456)
    N, D = 10, 2
    x = rng.standard_normal(N)
    X = rng.standard_normal((D, N))
    DX = m.ColVecs(X)
    DxX = m.BlockData([x, DX])
    assert len(DxX) == 2 * N                                    # :12-13
    assert DxX == DxX and DxX == m.BlockData([x, DX])           # :14-15
    assert len([v for v in DxX]) == 2 * N                       # :16
    assert DxX[0] == x[0] and DxX[1] == x[1] and DxX[N - 1] == x[N - 1]   # :17-19 (1-based there)
    assert np.array_equal(DxX[N], DX[0])                        # :20
    assert np.array_equal(DxX.view(1, 0), DX[0])                # :21
    assert np.array_equal(DxX.view(1, N - 1), DX[N - 1])        # :22
    idx = DxX.eachindex()                                       # :23-24  mortar([1:N, N+1:2N])
    assert np.array_equal(idx[0], np.arange(1, N + 1)) and np.array_equal(idx[1], np.arange(N + 1, 2 * N + 1))
    it = [v for v in DxX]                                       # :27-30
    assert it[0] == x[0] and it[N - 1] == x[-1]
    assert np.array_equal(it[N], DX[0]) and np.array_equal(it[-1], DX[N - 1])
    assert m.BlockData(x, DX) == DxX                            # :39


def test_blockdata_locate_walk(m):
    bd = m.BlockData(np.arange(3.0), np.arange(0.0), np.arange(5.0), np.arange(1.0))
    assert len(bd) == 9
    expect = [(0, 0), (0, 1), (0, 2), (2, 0), (2, 1), (2, 2), (2, 3), (2, 4), (3, 0)]
    assert [bd.locate(i) for i in range(9)] == expect           # empty block skipped like :71-78


def test_vcat_gpppinput(m):
    rng = np.random.default_rng(1)
    x, X = rng.standard_normal(10), rng.standard_normal((2, 10))
    ax, bx = m.GPPPInput("a", x), m.GPPPInput("b", m.ColVecs(X))
    v = m.vcat(ax, bx)                                          # :42-48
    assert isinstance(v, m.BlockData)
    flat = list(ax) + list(bx)
    assert len(v) == len(flat)
    for a, b in zip(v, flat):
        assert a[0] == b[0] and np.array_equal(a[1], b[1])
    assert ax[2] == ("a", x[2])


def test_eltype_rules(sb):
    rng = np.random.default_rng(0)
    DX = sb.ColVecs(rng.standard_normal((2, 4)))
    assert sb.BlockData([rng.standard_normal(5), rng.standard_normal(4)]).eltype() == ("scalar", np.dtype("float64"))  # :33
    assert sb.BlockData([rng.standard_normal(5), DX]).eltype() == ("any", None)                                        # :34
    assert sb.BlockData([DX, DX]).eltype()[0] == "vec"                                                                 # :35


def test_split_exact(m):
    rng = np.random.default_rng(2)
    x = m.BlockData(rng.standard_normal(5), rng.standard_normal(4))
    Y = rng.standard_normal((9, 3))
    Y1, Y2 = m.split(x, Y)
    assert np.array_equal(Y1, Y[0:5, :]) and np.array_equal(Y2, Y[5:, :])   # doctest gppp.jl:90-102
    y1, y2 = m.split(x, Y[:, 0])
    assert y1.shape == (5,) and y2.shape == (4,) and np.array_equal(y2, Y[5:, 0])
    with pytest.raises(RuntimeError, match=r"Expected length\(x\) == length\(y\)"):
        m.split(x, rng.standard_normal(8))
    with pytest.raises(RuntimeError, match=r"Expected length\(x\) == size\(Y, 1\)"):
        m.split(x, rng.standard_normal((8, 2)))


def test_block_ranges_ragged_config5(sb, orc):
    lens = (52429, 52429, 52429, 52429, 52428)                   # SURVEY 8d config 5
    bd = sb.BlockData(*[np.zeros(n) for n in lens])
    r = bd.block_ranges()
    assert r == [(1, 52429), (52430, 104858), (104859, 157287), (157288, 209716), (209717, 262144)]
    assert r == orc.get_indices(orc.BlockData(*[np.zeros(n) for n in lens]))
    assert bd.locate(52429) == (1, 0) and bd.locate(262143) == (4, 52427)
