"""SSR_UNet.restore_batch / GSR_UNet.restore_batch host logic with a stub engine: the clips are packed into one call in order,
the result comes back as one view per clip, and bad arguments raise before anything is called."""
import pytest
import torch


class StubEngine:
    device = torch.device("cpu")
    loaded = True

    def __init__(self):
        self.calls = []

    def ssr_restore_varlen(self, packed, lengths):
        self.calls.append((packed.clone(), list(lengths)))
        return packed * 0.5


def _model(cls_name="SSR_UNet"):
    import voicefixer_main_b200 as pkg
    m = getattr(pkg, cls_name)()
    m._eng = StubEngine()
    return m


@pytest.mark.parametrize("cls_name", ["SSR_UNet", "GSR_UNet"])
def test_ssr_restore_batch_packs_in_order_and_splits_into_views(cls_name):
    m = _model(cls_name)
    clips = [torch.arange(n, dtype=torch.float32) - 7 * i for i, n in enumerate([1025, 5000, 2048, 1100])]
    out = m.restore_batch(clips)
    (packed, lengths), = m._eng.calls
    assert lengths == [1025, 5000, 2048, 1100]
    assert torch.equal(packed, torch.cat(clips))
    assert [o.shape for o in out] == [c.shape for c in clips]
    for o, c in zip(out, clips):
        assert torch.equal(o, c * 0.5)
    assert all(o.untyped_storage().data_ptr() == out[0].untyped_storage().data_ptr() for o in out)   # views of one output


@pytest.mark.parametrize("bad, exc", [
    ([], ValueError),                                                        # empty list
    ((), ValueError),
    ("not a list", ValueError),
    ([torch.zeros(2000), "not a tensor"], ValueError),
    ([torch.zeros(1, 2000)], ValueError),                                    # not 1-D
    ([torch.zeros(2000), torch.zeros(1024)], ValueError),                    # too short for the reflect padding
    ([torch.zeros(2000, dtype=torch.float16)], TypeError),                   # dtype
    ([torch.zeros(2000), torch.zeros(2000, device="meta")], TypeError),      # device
])
def test_ssr_restore_batch_rejects_bad_arguments_before_calling(bad, exc):
    m = _model()
    with pytest.raises(exc):
        m.restore_batch(bad)
    assert m._eng.calls == []


def test_ssr_restore_batch_needs_a_device():
    from voicefixer_main_b200 import SSR_UNet
    with pytest.raises(RuntimeError):
        SSR_UNet().restore_batch([torch.zeros(2000)])
