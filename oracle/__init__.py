"""CPU restatements of the reference's algorithms -- TEST INFRASTRUCTURE ONLY.

Nothing under `end2end-asr-pytorch_b200/` imports this package and there is no CPU execution path in the product (it fails
loudly without the CUDA library and an H100).  The only importers are `tests/` (incl. the `tests/parity_cfg2.py` sweep),
`__graft_entry__.smoke()` and the CPU arms of `bench.py` (`cpu_baseline`, `--impl reference`).

* `asr_oracle.py`      -- the training hot path (front ends, encoder / decoder, loss, greedy search, Noam + Adam), pinned by
                          fixtures generated from the live reference (`tests/golden/`, `tests/test_oracle_golden.py`).
* `features_oracle.py` -- the audio feature front end (librosa.stft definition); unpinned against librosa (absent), pinned
                          against torch.stft (`tests/test_features.py`).
"""
