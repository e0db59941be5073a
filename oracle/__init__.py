"""CPU oracle for the community-1 diarization hot path.

TEST INFRASTRUCTURE ONLY.  This package is a CPU restatement (PyTorch CPU fp32 /
numpy fp64 / scipy) of the reference algorithm on the path named by
BASELINE.json.north_star.  Only ``tests/``, ``__graft_entry__.smoke()`` and
``bench.py``'s ``cpu_baseline`` / ``--impl reference`` legs may import it, and
only as the checker or as the timed CPU baseline -- never as the product.  The
product package (``pyannote_audio_b200``) must not import anything from here
and fails loudly when its CUDA library is missing.

Parity pinning status:

* StatsPool, Powerset, VBx/PLDA, ResNet34 trunk, receptive-field arithmetic:
  PINNED -- validated in the build container against the reference's own files
  loaded by path (``oracle/ref_loader.py``) and against the reference's golden
  vectors (tests/test_stats_pool.py, tests/utils/test_powerset.py,
  tests/test_clustering.py); committed fixtures in ``tests/golden/``.
* kaldi fbank, nn.LSTM, scipy linkage/fcluster/cdist/linear_sum_assignment:
  the oracle calls the very same third-party code the reference calls.
* SincNet filter bank (asteroid-filterbanks 0.4.0 ``ParamSincFB``) and
  pyannote.core 6.0.1 frame arithmetic (``SlidingWindow.closest_frame`` /
  ``crop``): sources are absent from /root/reference and not installed;
  restated from the published algorithm -- PARITY UNPINNED for those two
  pieces (shape facts from the reference tutorials are checked).
"""
