"""Labels of the problem's children (basics/optilayer.py OptiChild._make_label): the reference's rule,
for as many children as a process creates."""
from omg_tools_b200.basics.optilayer import OptiChild


def test_labels_take_the_first_free_index_past_the_recursion_limit():
    """With 3000 obstacles and a few vehicles labelled already, the next obstacle is obstacle3000 and a
    vehicle asked for as vehicle1 skips the taken indices; an unlabelled prefix starts at 0.  (The
    reference's recursive search, one call per taken index, raises RecursionError here.)"""
    saved = list(OptiChild._labels)
    try:
        OptiChild._labels[:] = ['obstacle%d' % k for k in range(3000)] + ['vehicle0', 'vehicle1', 'vehicle2']
        assert OptiChild._make_label('obstacle') == 'obstacle3000'
        assert OptiChild._make_label('obstacle') == 'obstacle3001'
        assert OptiChild._make_label('obstacle2999') == 'obstacle3002'
        assert OptiChild._make_label('vehicle1') == 'vehicle3'
        assert OptiChild._make_label('p2p') == 'p2p0'
        assert OptiChild._make_label('veh007') == 'veh007'
        assert OptiChild._make_label('veh007') == 'veh8'
    finally:
        OptiChild._labels[:] = saved
