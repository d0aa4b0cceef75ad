"""`get` on device PCM of several chunks queues the approx search of chunk k + 1 before chunk k's selection, refine and decode
(awm_sync_approx_enqueue, two approx slots); host PCM and several keys keep the serial chunk loop (AWM_TRACE shows which ran).  Both loops must give the same
`--json` document, pattern for pattern: the same audio as a device float buffer (pipelined) and as a pinned 16 bit host buffer
(serial).  The float values are the 16 bit samples * 2^-15, exactly what the 16 bit path converts them to on the device."""
import json

import pytest

from audiowmark_b200 import hostapi as H

pytestmark = pytest.mark.gpu

RATE = 44100
PAYLOAD = "0123456789abcdef0011223344556677"
KEY2 = bytes(range(1, 17))


def marked(minutes):
    """noise at -6 dBFS marked with PAYLOAD under the default key, as (device float32 tensor, pinned int16 tensor)"""
    import torch
    n, ch = int(minutes * 60 * RATE), 2
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev)
    g.manual_seed(7)
    x = torch.rand((n, ch), device=dev, generator=g, dtype=torch.float32) - 0.5
    y = torch.empty_like(x)
    torch.cuda.synchronize()               # the library works on its own stream
    H.add(x.data_ptr(), PAYLOAD, None, y.data_ptr(), n, ch)
    torch.cuda.synchronize()
    y16 = torch.floor(y * 32768.0).clamp_(-32768, 32767).to(torch.int16)
    del x, y
    host16 = torch.empty(y16.shape, dtype=torch.int16, pin_memory=True)
    host16.copy_(y16)
    yf = y16.to(torch.float32) / 32768.0
    torch.cuda.synchronize()
    return yf, host16


def queued_ahead(capfd):
    """number of approx searches the last `get` queued ahead of their chunk (AWM_TRACE lines on stderr)"""
    return capfd.readouterr().err.count("queued ahead")


# (minutes, keys, searches queued ahead on device input): 3 chunks for 1 h and for 65 min; several keys keep the serial loop
@pytest.mark.parametrize("minutes,keys,ahead", [(60.0, [None], 2), (65.0, [None], 2), (60.0, [None, KEY2], 0)],
                         ids=["1h", "65min_short_last_chunk", "1h_two_keys_serial"])
def test_pipelined_get_equals_serial(minutes, keys, ahead, capfd, monkeypatch):
    H.set_params()
    yf, host16 = marked(minutes)
    n, ch = yf.shape
    key_bytes = [k or bytes(16) for k in keys]
    monkeypatch.setenv("AWM_TRACE", "1")
    capfd.readouterr()
    doc_dev = json.loads(H.get(yf.data_ptr(), keys=key_bytes, n_frames=n, channels=ch, parse=False))
    assert queued_ahead(capfd) == ahead
    doc_host = json.loads(H.get_s16(host16.numpy(), keys=key_bytes, parse=False))
    assert queued_ahead(capfd) == 0                      # host PCM: serial loop
    monkeypatch.delenv("AWM_TRACE")
    assert doc_dev == doc_host
    real = [m for m in doc_dev["matches"] if m["quality"] > 0.35]
    assert len(real) > 50 and all(m["bits"] == PAYLOAD for m in real)
    # the same device buffer again: the approx slots are reused
    assert json.loads(H.get(yf.data_ptr(), keys=key_bytes, n_frames=n, channels=ch, parse=False)) == doc_dev
