"""audiolazy_b200 -- H100-native implementation of AudioLazy's linear-filter hot path.

Same names as the reference (``from audiolazy import ...``) for everything on the path:
``Stream``, ``thub``, ``Poly``, ``ZFilter``, ``z``, ``LinearFilter``, ``CascadeFilter``,
``ParallelFilter``, ``comb``, ``resonator``, ``lowpass``, ``highpass``, ``erb``,
``gammatone``, ``gammatone_erb_constants``, ``sHz``, ``almost_eq``; plus the bank object
the reference lacks (``FilterBank``, ``gammatone_bank``, ``erb_space``); ``amdf`` with its batched
form ``AmdfBank`` (many streams x many lags) and the ``freq2lag`` / ``lag2freq`` converters; ``zcross`` with its
batched form ``Zcross`` (flags or per-block counts of many streams); ``lpc_frames`` with its batched form ``LpcFrames``
(``lpc.kautocor`` or ``lpc.kcovar`` of every block of many streams); ``window`` / ``wsymm``, ``overlap_add`` and
``stft`` with their batched forms ``OverlapAdd`` and ``Stft`` (short-time Fourier analysis, resynthesis and
overlap-add of many streams); ``lagrange`` and ``resample`` with its batched form ``Resampler`` (Lagrange sample-rate
conversion of many streams); ``dft`` at arbitrary frequencies with its batched form ``Dft`` and the lazy ``dft_frames``
(the DFT of every frame of many streams); ``unwrap`` and ``clip`` with their batched forms ``Unwrap`` (phase unwrapping
of many streams, carried block by block) and ``Clip``; ``parcor`` with its batched form ``parcor_batch`` (the
reflection coefficients and ``parcor_stable`` of many LPC rows, such as ``LpcFrames``' output); ``LpcFilter`` (the
residual of many streams through their frame-wise LPC analysis filters, and its all-pole resynthesis).

The per-sample recurrences run in hand-written sm_90a CUDA kernels behind the C ABIs of
``include/alz_b200.h``, ``include/alz_b200_amdf.h``, ``include/alz_b200_zcross.h``, ``include/alz_b200_lpc.h``, ``include/alz_b200_stft.h``, ``include/alz_b200_resample.h``, ``include/alz_b200_dft.h``, ``include/alz_b200_unwrap.h``, ``include/alz_b200_parcor.h`` and ``include/alz_b200_lpcfilt.h``; importing this package does not need a GPU, calling a filter does.
"""
from .core import StrategyDict
from .stream import Stream, StreamTeeHub, thub, tostream, avoid_stream
from .misc import sHz, almost_eq, zero_pad, elementwise, freq2lag, lag2freq, DEFAULT_SAMPLE_RATE
from .poly import Poly, x
from .filters import (LinearFilterProperties, LinearFilter, ZFilter, z, FilterList, CascadeFilter, ParallelFilter,
                      comb, resonator, lowpass, highpass)
from .auditory import erb, gammatone, gammatone_erb_constants, erb_space, gammatone_bank
from .bank import FilterBank, BankState
from .callers import envelope, maverage, karplus_strong, accumulate_z, zeros, ones, impulse, white_noise
from .analysis import amdf, AmdfBank, AmdfState
from .crossing import zcross, Zcross, ZcrossState
from .io import chunks, WavStream, wav_batch, pcm_to_float32
from .linear_prediction import (ParCorError, acorr, lag_matrix, toeplitz, levinson_durbin, lpc, parcor, parcor_stable,
                                lsf, lsf_stable, LpcFrames, LpcState, lpc_frames, parcor_batch, ParcorResult,
                                LpcFilter, LpcFilterState)
from .spectral import window, wsymm, overlap_add, stft, OverlapAdd, OlaState, Stft, StftState
from .resampling import lagrange, resample, Resampler, ResampleState
from .fourier import dft, Dft, DftState, dft_frames
from .unwrapping import unwrap, Unwrap, UnwrapState, clip, Clip

__version__ = "0.1.0"
