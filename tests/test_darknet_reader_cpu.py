"""The .weights reader refuses cfgs whose layers load_weights would partly skip (dontload, dontloadscales): the reference
then keeps those layers' random initial parameters, which no file describes."""
import os

import pytest

from image_b200 import darknet as dn
from oracle import ref_darknet as rd

pytestmark = pytest.mark.skipif(not rd.have_ref(), reason="reference build oracle/_ref/libref_darknet.so absent")


@pytest.mark.parametrize("option", ["dontload", "dontloadscales"])
def test_layers_that_skip_their_weights_are_refused(tmp_path, option):
    src = open(rd.path("tiny.cfg")).read()
    cfg = os.path.join(str(tmp_path), "tiny.cfg")
    open(cfg, "w").write(src.replace("[convolutional]\n", "[convolutional]\n%s=1\n" % option, 1))
    net = dn.parse_cfg(cfg)
    with pytest.raises(ValueError, match=option):
        dn.read_weights(rd.path("tiny.weights"), net)
