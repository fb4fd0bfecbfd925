"""The batch-1 step of the persistent MLP kernel (csrc/mlp_v2.cuh, variants 3 / 5 / 6) issues the rank-1 updates of layer 1
and of the head at the top of the following step instead of at the end of their own (docs/KERNELS.md §2).  That only
moves instructions: every weight receives the same FMAs on the same operands.  These fingerprints were taken from the
kernel source before the move (SIMT build on the CPU, csrc/host_shim.h), so any change in the bits of the trained model
or of the reported losses fails here — including at the chunk boundaries, where the pending updates are flushed: 97 x 2
epochs ends on a 2-step chunk, 150 steps of 200 on a 22-step chunk, 65 samples on a 1-step chunk."""
import hashlib

import pytest
import torch

from colearn_federated_learning_b200.models import build_model, flatten_params

NETS = {0: ("ffnn", (10, 50, 30, 10, 1), ("bce", "sse", "mse")), 1: ("mlp", (10, 64, 64, 2), ("xent",)),
        2: ("testing_remote", (2, 50, 10, 1), ("sse", "mse"))}
LOSS_CODES = {"bce": 0, "sse": 1, "xent": 2, "mse": 3}
SIZES = {97: (2, -1), 200: (1, 150), 65: (1, -1)}   # n: (epochs, max_steps)

# "<net>-<loss>-v<variant>-n<n>": (sha256 of the trained parameters, sha256 of the [last, mean] losses), first 32 hex digits
FINGERPRINTS = {
    "ffnn-bce-v5-n97": ("b38834ed49f02f305ec6943afd16e848", "212717896d20646f5657d1bb1852b123"),
    "ffnn-bce-v5-n200": ("73274ba2abaa23f62dc7238be62e164c", "4733b34a7e59a2e4112b8fdf6a813c02"),
    "ffnn-bce-v5-n65": ("21b73d6f3fb7d0f66e26f8be4e37f1c9", "75b27df17d52a4bcd2d15b48c0181690"),
    "ffnn-bce-v6-n97": ("b38834ed49f02f305ec6943afd16e848", "212717896d20646f5657d1bb1852b123"),
    "ffnn-bce-v6-n200": ("73274ba2abaa23f62dc7238be62e164c", "4733b34a7e59a2e4112b8fdf6a813c02"),
    "ffnn-bce-v6-n65": ("21b73d6f3fb7d0f66e26f8be4e37f1c9", "75b27df17d52a4bcd2d15b48c0181690"),
    "ffnn-bce-v3-n97": ("7a872e337a45d0fd3082eab48e1a796b", "212717896d20646f5657d1bb1852b123"),
    "ffnn-bce-v3-n200": ("03c26b066e4480b467cd662fe33c1e09", "aa26e3b4c3929799486d74ab7eefdf3e"),
    "ffnn-bce-v3-n65": ("8d47587d64a5237fe95471d73801dc49", "75b27df17d52a4bcd2d15b48c0181690"),
    "ffnn-sse-v5-n97": ("2711210c2e135a1095f39c31078ad600", "3e2ed348f3dc210042ddaf6331bf4dac"),
    "ffnn-sse-v5-n200": ("c2471d7f07a66eda3c7d76159b16ed46", "6147528ff796b9e8eac54457c1422311"),
    "ffnn-sse-v5-n65": ("0bd6bf07661fc2277f997e0f27484abe", "58c439a7b56c28f2e6c9eb77625d33f0"),
    "ffnn-sse-v6-n97": ("2711210c2e135a1095f39c31078ad600", "3e2ed348f3dc210042ddaf6331bf4dac"),
    "ffnn-sse-v6-n200": ("c2471d7f07a66eda3c7d76159b16ed46", "6147528ff796b9e8eac54457c1422311"),
    "ffnn-sse-v6-n65": ("0bd6bf07661fc2277f997e0f27484abe", "58c439a7b56c28f2e6c9eb77625d33f0"),
    "ffnn-sse-v3-n97": ("5a331fb7f664d3f0bc6aea90db987c2d", "de003fef160c6e7c6ab402acdb420046"),
    "ffnn-sse-v3-n200": ("929d3e3fe4cbf30fa87109c181ba382c", "6147528ff796b9e8eac54457c1422311"),
    "ffnn-sse-v3-n65": ("8b9bf453e72b14a3c016406e6bcf2f7c", "58c439a7b56c28f2e6c9eb77625d33f0"),
    "ffnn-mse-v5-n97": ("4ce537e7edadd34464fbbe72c9d01236", "679fb67bfdab14674e54ac15b858f58e"),
    "ffnn-mse-v5-n200": ("a1d900ed948f023cca9a662523a4b99d", "daf0e921baf043fb8e875957f765fe49"),
    "ffnn-mse-v5-n65": ("d57674a44aba3803ce2bdeb9cf67f52e", "2f12327cef416d6376e02c49ff285707"),
    "ffnn-mse-v6-n97": ("4ce537e7edadd34464fbbe72c9d01236", "679fb67bfdab14674e54ac15b858f58e"),
    "ffnn-mse-v6-n200": ("a1d900ed948f023cca9a662523a4b99d", "daf0e921baf043fb8e875957f765fe49"),
    "ffnn-mse-v6-n65": ("d57674a44aba3803ce2bdeb9cf67f52e", "2f12327cef416d6376e02c49ff285707"),
    "ffnn-mse-v3-n97": ("fe02b0eb25e2ecc47e152a21cc055787", "e7a583218c6d8f9410f297bbeff74eef"),
    "ffnn-mse-v3-n200": ("08b8db23afcf8f4f17b7a6ea14bbf9bf", "daf0e921baf043fb8e875957f765fe49"),
    "ffnn-mse-v3-n65": ("ee84d183f6f6f389cc836faa9d7ee4cd", "2f12327cef416d6376e02c49ff285707"),
    "mlp-xent-v5-n97": ("86a96da6d40d5dd3208c0b3cbd2b54ef", "a15abdbca20df8e52677a3e5a7836b43"),
    "mlp-xent-v5-n200": ("327ae17c373fae1e32ab516157e62050", "6d827f7037749915e13c49d8f7f7131f"),
    "mlp-xent-v5-n65": ("bfb7e49699a55a74270909255e1f5856", "f54df052f5d86da01aff6718882ac4b5"),
    "mlp-xent-v6-n97": ("86a96da6d40d5dd3208c0b3cbd2b54ef", "a15abdbca20df8e52677a3e5a7836b43"),
    "mlp-xent-v6-n200": ("327ae17c373fae1e32ab516157e62050", "6d827f7037749915e13c49d8f7f7131f"),
    "mlp-xent-v6-n65": ("bfb7e49699a55a74270909255e1f5856", "f54df052f5d86da01aff6718882ac4b5"),
    "mlp-xent-v3-n97": ("be09a7c8e3db0b62649df70ca003727d", "773d641bd881293a225e2a216eee905e"),
    "mlp-xent-v3-n200": ("85a5ac5ccc9cabd92cb79b24d928b089", "5c63cb9b7322c5c5232b420afe515214"),
    "mlp-xent-v3-n65": ("de1e334aa5f5a33437ca4fd7803d5ed8", "d5c33712e84651862f3cbdb5b8d4ffc5"),
    "testing_remote-sse-v5-n97": ("3862f38bf61453e2b61611768400b572", "04dcfc540c9bca08388fbc4d9472e865"),
    "testing_remote-sse-v5-n200": ("dd36a77489e70615f1a3ad14d68b9834", "294804c8f2dddd70aff0c1ac7652af5a"),
    "testing_remote-sse-v5-n65": ("3494c4cd3ae3c888654d0085b6da7955", "acd4300049fd526512e24f5f1dc8f74d"),
    "testing_remote-sse-v6-n97": ("3862f38bf61453e2b61611768400b572", "04dcfc540c9bca08388fbc4d9472e865"),
    "testing_remote-sse-v6-n200": ("dd36a77489e70615f1a3ad14d68b9834", "294804c8f2dddd70aff0c1ac7652af5a"),
    "testing_remote-sse-v6-n65": ("3494c4cd3ae3c888654d0085b6da7955", "acd4300049fd526512e24f5f1dc8f74d"),
    "testing_remote-sse-v3-n97": ("ddfcc86d8b74436c90f15835065b20c6", "a849b62699ea1718d7391c2e597a010e"),
    "testing_remote-sse-v3-n200": ("3be79e5c084f733933bcff70b6d5acd6", "6a7234b75ca31bb414a914eb07ceddba"),
    "testing_remote-sse-v3-n65": ("244e8ea92b03de7ce58a7e7fe59d7dcd", "5c3ed434fb32fe2e4cccaa0e373d681d"),
    "testing_remote-mse-v5-n97": ("4c1b5d5971c75964a21014c7af839dc4", "d058905fa0679ef15b012967ea390bcc"),
    "testing_remote-mse-v5-n200": ("fcfc47473936ed1710857cf2544022c7", "f1c6d839b3523770c39f21aebac5910e"),
    "testing_remote-mse-v5-n65": ("ec87279d690e58937b02273d3cc7d185", "b47d5405042322b1c8aa4762dcfba24a"),
    "testing_remote-mse-v6-n97": ("4c1b5d5971c75964a21014c7af839dc4", "d058905fa0679ef15b012967ea390bcc"),
    "testing_remote-mse-v6-n200": ("fcfc47473936ed1710857cf2544022c7", "f1c6d839b3523770c39f21aebac5910e"),
    "testing_remote-mse-v6-n65": ("ec87279d690e58937b02273d3cc7d185", "b47d5405042322b1c8aa4762dcfba24a"),
    "testing_remote-mse-v3-n97": ("48ed434591509536ec5cdf3068e8a7ee", "cc857d9c1f85ea51bffcef8ef5d3c303"),
    "testing_remote-mse-v3-n200": ("e6a81329b28a7128c6a73777f01a0f61", "13b3f0bb1fa2d9570f799724fda409c5"),
    "testing_remote-mse-v3-n65": ("add55bb5ada5344a2ba243d0774d194e", "b47d5405042322b1c8aa4762dcfba24a"),
}


@pytest.fixture(scope="module")
def simt():
    import importlib.util
    import os
    import shutil

    from colearn_federated_learning_b200.ops import build
    if shutil.which("g++") is None or not os.path.exists(os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include", "cuda_runtime.h")):
        pytest.skip("no g++ / CUDA headers on this box: the SIMT emulator cannot be built")
    path = build.build_simt_emul()
    spec = importlib.util.spec_from_file_location("_colearn_simt", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("case", sorted(FINGERPRINTS))
def test_batch1_step_order_keeps_bits(simt, case):
    name, loss, variant, n = case.split("-")
    kind = next(k for k, v in NETS.items() if v[0] == name)
    dims = NETS[kind][1]
    variant, n = int(variant[1:]), int(n[1:])
    epochs, max_steps = SIZES[n]
    g = torch.Generator().manual_seed(1000 + kind * 10 + LOSS_CODES[loss])
    x = torch.rand(n, dims[0], generator=g)
    y = (torch.randint(0, dims[-1], (n, 1), generator=g).float() if loss == "xent"
         else (torch.rand(n, dims[-1], generator=g) > 0.5).float())
    torch.manual_seed(kind)
    flat0 = flatten_params(build_model(name)).clone()
    got = flat0.clone()
    losses = simt.mlp_local_sgd(kind, flat0, [got], [x], [y], [None], 1, epochs, max_steps, LOSS_CODES[loss], 0.05, variant, [1.0],
                                False, None, perm_seed=12345, perm_row0=0,
                                perm_scratch=torch.full((1, epochs * n), -1, dtype=torch.int32))
    want_model, want_losses = FINGERPRINTS[case]
    assert hashlib.sha256(got.numpy().tobytes()).hexdigest()[:32] == want_model
    assert hashlib.sha256(losses.numpy().tobytes()).hexdigest()[:32] == want_losses
