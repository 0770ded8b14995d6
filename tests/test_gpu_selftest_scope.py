"""The vf_selftest_* hooks leave the engine as they found them.  A case packs weights into the context, allocates buffers
and may fail half way; the engine's cached plans, weights, options and launch count must not show it afterwards, whichever
way the case ended."""
import pytest
import torch

import test_gpu_analysis as AN
import test_gpu_aux as AUX
import test_gpu_layers as LAY
from oracle import analysis as A
from oracle import vf_oracle as O
from voicefixer_main_b200 import _lib as VL

pytestmark = pytest.mark.gpu

N = 13230                     # samples per clip of the restores around the cases: 31 frames


def test_cases_leave_the_engine_as_they_found_it():
    from voicefixer_main_b200.model import Engine
    from voicefixer_main_b200.weights import make_state
    e = Engine("cuda:0")
    try:
        e.load_state(make_state(1234))
        wav = O.synth_clips(2, N, seed=3).cuda()
        e.workspace_bytes(2, N)
        want = e.restore(wav).cpu()           # the plans these calls use are built and cached here
        ws, cache = e.workspace_bytes(2, N), e.plan_cache_info()
        n0 = e.launch_count()

        # a layer rejected after its weights were packed: the loaders' packer takes N = 48, Builder::gemm does not
        bad = LAY.build(LAY.C("scope.cout48", LAY.CONV1D, L=64, cin=64, cout=48, k=3))
        with pytest.raises(VL.EngineError) as ei:
            e.selftest_layer(bad.lc)
        assert ei.value.code == VL.VF_EINVAL and "N=48 not a multiple of 32" in str(ei.value)

        # a layer, one launch
        LAY.run_and_check(e, LAY.BY_NAME["conv1.mel_l0"])

        # a tail case, which packs the tail weights: the peak memset and the tail conv
        name = "tail.L300_lt_one_tile"
        args = AUX.tail_case(name, AUX.TAIL_CASES[name], 1, 1)
        e.selftest_op(args[0].oc)
        e.check_errors()
        AUX.check_tail(name, *args, 1, 1)

        # a GRU layer, one launch
        lengths, T = [16, 5], 16
        G, w, b = AN._gru_inputs(len(lengths), T, seed=5)
        got, G, w, b = AN._run_gru(e, G, w, b, lengths, False, T)
        AN._check_gru(got, A.gru_layer(G, w, b, lengths), lengths, T)
        launches = e.launch_count() - n0

        # a plan sweep still runs, and launches nothing
        assert e.selftest_plan_gemms(0, 2, 101)
        # no weights or plan buffers left behind
        assert e.workspace_bytes(2, N) == ws
        assert e.plan_cache_info() == cache
        assert torch.equal(e.restore(wav).cpu(), want)
        assert launches == 1 + 2 + 1, launches
        e.check_errors()
    finally:
        e.close()
