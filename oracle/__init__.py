"""CPU oracle for the OLMoASR hot path -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this package.  Nothing under olmoasr_b200/ imports it; the product path raises when the CUDA
extension is missing instead of falling back to anything here.

Contents
  logmel.py    numpy restatement of whisper.audio.{pad_or_trim, mel_filters, log_mel_spectrogram}
               (openai-whisper, un-pinned dependency of the reference: requirements.txt:21; the
               docstrings of the reference cite upstream commit ba3f3cd5).  Pinned against
               transformers.WhisperFeatureExtractor (an independent implementation) in
               tests/golden/logmel_*.npz -- see tools/make_golden.py.
  model.py     torch-CPU restatement of olmoasr/model.py and olmoasr/inf_model.py (modules, init order,
               autocast rounding points).  Pinned against the UNMODIFIED reference files imported via
               ref_import.py in this container; golden outputs in tests/golden/model_*.pt.
  decoding.py  restatement of whisper.decoding's greedy path (DecodingTask / PyTorchInference /
               GreedyDecoder / SuppressBlank / SuppressTokens).  The upstream package is absent here, so
               the LOOP is "parity unpinned"; the model calls inside it are pinned through model.py.
  synth.py     the synthetic batch of SURVEY.md section 8(d).
  ref_import.py  imports olmoasr/{model,inf_model}.py unmodified behind three stub
               modules (only where OLMOASR_REFERENCE_ROOT names a reference checkout).
"""
