"""The fused trunk chains' warpgroups hand the activation buffer's halves to each other through per-half barriers and
drift apart by up to the weight ring's depth.  Those barriers count one phase per generation of the buffer, across the
layers and tiles a CTA walks, so the cases here make the phases wrap many times: grids of 1 and 3 CTAs over many tiles,
both network depths (an odd and an even number of generations per tile), M not a multiple of 64, device row counts with
tiles past the live rows, 1 and 3 passes, and every or only the last activations kept.  The fused runs must write the
bytes the layer-by-layer GEMMs write (the span forward's instantiation is checked through the training step's span
tests)."""
import pytest
import torch

import test_tc_dgrad_chain as dg
import test_tc_trunk_chain as fw

pytestmark = pytest.mark.gpu

CAP = 1000      # 16 row tiles of 64: one CTA walks all of them, three CTAs 5 or 6 each


@pytest.mark.parametrize("rows", [None, 999, 333, 0])
@pytest.mark.parametrize("prec", ["f16x3", "f16x1", "bf16x3"])
@pytest.mark.parametrize("name", list(fw.NETS))
@pytest.mark.parametrize("max_ctas", [1, 3])
def test_forward_chain_drift(max_ctas, name, prec, rows):
    net = fw._net(name, CAP, 17 * max_ctas + len(name) + len(prec))
    nt = net[0]
    for outputs in (None, 3 << (nt - 2)):
        ref = fw._run(net, CAP, prec, 0, outputs=outputs, rows=rows)
        fw._same(fw._run(net, CAP, prec, 1, max_ctas=max_ctas, outputs=outputs, rows=rows), ref)


@pytest.mark.parametrize("rows", [None, 999, 333, 0])
@pytest.mark.parametrize("prec", list(dg.PRECS))
@pytest.mark.parametrize("name", list(dg.NETS))
@pytest.mark.parametrize("max_ctas", [1, 3])
def test_dgrad_chain_drift(max_ctas, name, prec, rows):
    """Integer gradients through signed permutations: the column sums are exact in any order, so they must match too."""
    inp = dg._inputs(name, CAP, 23 * max_ctas + len(name) + len(prec), ints=True)
    ref = dg._run(inp, CAP, prec, 0, rows=rows)
    dg._same(dg._run(inp, CAP, prec, 1, max_ctas=max_ctas, rows=rows), ref, exact_sums=True)
