"""The fused trunk chains on 128-row tiles, each consumer warpgroup on its own 64 rows of a tile: a tile whose second
warpgroup has no live row (M mod 128 in 1 ... 64, or a device row count that ends inside the first warpgroup's rows)
still streams and releases every weight stage and writes its 128-row image tiles whole.  At 1 and 3 CTAs (the weight
ring wraps across tiles), both network depths and 1 and 3 passes, the chains must write the bytes the layer-by-layer
GEMMs write, through the same self-tests as test_tc_trunk_chain.py and test_tc_dgrad_chain.py."""
import pytest

import test_tc_dgrad_chain as dg
import test_tc_trunk_chain as fw

pytestmark = pytest.mark.gpu

ROWS = [129, 192, 641]          # 1, 64 and 1 live rows in the last tile
CAP, COUNTS = 300, [1, 64, 129, 192, 257]    # device row counts of a 300-row capacity, all inside a first warpgroup


@pytest.mark.parametrize("max_ctas", [1, 3])
@pytest.mark.parametrize("prec", ["f16x3", "f16x1"])
@pytest.mark.parametrize("name", list(fw.NETS))
@pytest.mark.parametrize("M", ROWS)
def test_forward_idle_warpgroup(M, name, prec, max_ctas):
    net = fw._net(name, M, 13 * M + max_ctas)
    fw._same(fw._run(net, M, prec, 1, max_ctas=max_ctas), fw._run(net, M, prec, 0))


@pytest.mark.parametrize("max_ctas", [1, 3])
@pytest.mark.parametrize("name", list(fw.NETS))
@pytest.mark.parametrize("K", COUNTS)
def test_forward_device_rows(K, name, max_ctas):
    net = fw._net(name, CAP, 5 * K + max_ctas)
    fw._same(fw._run(net, CAP, "f16x3", 1, max_ctas=max_ctas, rows=K), fw._run(net, CAP, "f16x3", 0, rows=K))


@pytest.mark.parametrize("rows", [None, 130])
@pytest.mark.parametrize("name", list(fw.NETS))
def test_forward_bits_idle_warpgroup(name, rows):
    dg.test_forward_chain_bits(192 if rows is None else CAP, name, rows)


@pytest.mark.parametrize("max_ctas", [1, 3])
@pytest.mark.parametrize("prec", list(dg.PRECS))
@pytest.mark.parametrize("name", list(dg.NETS))
@pytest.mark.parametrize("M", ROWS)
def test_dgrad_idle_warpgroup(M, name, prec, max_ctas):
    """Small-integer gradients through signed permutations, so the column sums are exact in any order."""
    inp = dg._inputs(name, M, 11 * M + max_ctas, ints=True)
    dg._same(dg._run(inp, M, prec, 1, max_ctas=max_ctas), dg._run(inp, M, prec, 0), exact_sums=True)


@pytest.mark.parametrize("max_ctas", [1, 3])
@pytest.mark.parametrize("name", list(dg.NETS))
@pytest.mark.parametrize("K", COUNTS)
def test_dgrad_device_rows(K, name, max_ctas):
    inp = dg._inputs(name, CAP, 7 * K + max_ctas, ints=True)
    dg._same(dg._run(inp, CAP, "bf16x3", 1, max_ctas=max_ctas, rows=K), dg._run(inp, CAP, "bf16x3", 0, rows=K),
             exact_sums=True)
