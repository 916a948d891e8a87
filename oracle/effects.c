/* TEST INFRASTRUCTURE ONLY — CPU restatement of the reference's vocal effects stage, `add_audio_effects`
 * (src/main.py:206-226):
 *
 *     board = Pedalboard([HighpassFilter(), Compressor(ratio=4, threshold_db=-15),
 *                         Reverb(room_size=..., dry_level=..., wet_level=..., damping=...)])
 *     with AudioFile(in) as f, AudioFile(out, 'w', f.samplerate, f.num_channels) as o:
 *         while f.tell() < f.frames: o.write(board(f.read(int(f.samplerate)), f.samplerate, reset=False))
 *
 * `pedalboard==0.7.7` (requirements.txt:11) is a third-party dependency, absent from the reference repository; it
 * wraps JUCE 6 DSP classes.  Their published algorithms are restated below — PARITY UNPINNED (restated from the published
 * sources of pedalboard / JUCE; nothing here was executed against them):
 *
 *   AudioFile.read         16-bit WAV -> float: sample * 2^-15 (JUCE reads ints left-justified in 32 bits, * 1/0x7fffffff in float)
 *   HighpassFilter()       cutoff 50 Hz; juce::dsp::IIR::Coefficients<float>::makeFirstOrderHighPass:
 *                          n = tan(pi f / sr); (b0, b1, a0, a1) = (1, -1, n + 1, n - 1) / a0; transposed direct form II:
 *                          y = b0 x + s; s = b1 x - a1 y (snapToZero of s once per processed block; Pedalboard.process
 *                          hands blocks of 8192 samples to the plugins)
 *   Compressor(4, -15 dB)  attack 1 ms, release 100 ms; juce::dsp::Compressor: env = BallisticsFilter(peak):
 *                          a = |y|; cte = a > env ? cteAT : cteRL; env = a + cte (env - a), cte = exp(-2 pi 1000 / sr / ms);
 *                          gain = env < thr ? 1 : pow(env / thr, 1 / ratio - 1), thr = 10^(dB / 20)
 *   Reverb(...)            juce::Reverb (Freeverb), mono: 8 parallel combs (tunings 1116..1617 at 44.1 kHz, scaled by the
 *                          integer sample rate), 4 series all-passes (556, 441, 341, 225; gain 0.5), input gain 0.015,
 *                          damp = damping * 0.4, feedback = room * 0.28 + 0.7, wet1 = 0.5 * (wet * 3) * (1 + width), dry * 2;
 *                          the smoothed parameters start at their targets (set before prepare()); JUCE_UNDENORMALISE
 *                          (x += 0.1f; x -= 0.1f) as on Intel builds
 *   AudioFile.write        float -> 16-bit WAV: juce::AudioFormatWriter::writeFromFloatArrays: int32 = x <= -1 ? INT_MIN :
 *                          x >= 1 ? INT_MAX : roundToInt(INT_MAX * (double) x) (round half even), the WAV writer keeps the
 *                          high 16 bits
 *
 * Build: gcc -O2 -ffp-contract=off -shared -fPIC (see oracle/build_c.py).  Mono only: the reference only ever feeds the RVC
 * output (mono) through this stage. */
#include <limits.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define UNDENORMALISE(x) \
  do {                   \
    (x) += 0.1f;         \
    (x) -= 0.1f;         \
  } while (0)

static const short COMB_TUNINGS[8] = {1116, 1188, 1277, 1356, 1422, 1491, 1557, 1617};
static const short ALLPASS_TUNINGS[4] = {556, 441, 341, 225};

typedef struct {
  float* buf;
  int size, idx;
  float last;
} delay_line;

static int line_init(delay_line* d, int size) {
  d->buf = (float*)calloc((size_t)size, sizeof(float));
  d->size = size;
  d->idx = 0;
  d->last = 0.0f;
  return d->buf != NULL;
}

/* stages (optional, may be NULL): [3][n] floats = after the high-pass, after the compressor, after the reverb */
int oracle_add_audio_effects_mono(const int16_t* in, int16_t* out, int64_t n, int sample_rate, float cutoff_hz,
                                  float threshold_db, float ratio, float attack_ms, float release_ms, float room_size,
                                  float damping, float wet_level, float dry_level, float width, int block, float* stages) {
  volatile float vf;
  /* ---- high-pass */
  const float nn = tanf((float)M_PI * cutoff_hz / (float)sample_rate);
  const float a0inv = 1.0f / (nn + 1.0f);
  const float b0 = 1.0f * a0inv, b1 = -1.0f * a0inv, a1 = (nn - 1.0f) * a0inv;
  float lv1 = 0.0f;
  /* ---- compressor */
  const float exp_factor = (float)(-2.0 * M_PI * 1000.0 / (double)sample_rate);
  const float cte_at = attack_ms < 1.0e-3f ? 0.0f : expf(exp_factor / attack_ms);
  const float cte_rl = release_ms < 1.0e-3f ? 0.0f : expf(exp_factor / release_ms);
  const float thr = threshold_db > -200.0f ? powf(10.0f, threshold_db * 0.05f) : 0.0f;
  const float thr_inv = 1.0f / thr, ratio_inv = 1.0f / ratio;
  float yold = 0.0f;
  /* ---- reverb */
  delay_line comb[8], ap[4];
  for (int j = 0; j < 8; ++j)
    if (!line_init(&comb[j], (sample_rate * COMB_TUNINGS[j]) / 44100)) return -1;
  for (int j = 0; j < 4; ++j)
    if (!line_init(&ap[j], (sample_rate * ALLPASS_TUNINGS[j]) / 44100)) return -1;
  const float gain = 0.015f;
  const float damp = damping * 0.4f, feedback = room_size * 0.28f + 0.7f;
  const float wet = wet_level * 3.0f, dry = dry_level * 2.0f;
  const float wet1 = 0.5f * wet * (1.0f + width);
  (void)vf;
  for (int64_t t = 0; t < n; ++t) {
    const float x = (float)((int32_t)in[t] << 16) * (1.0f / (float)0x7fffffff);
    /* IIR::Filter<float>, order 1 */
    const float y = x * b0 + lv1;
    lv1 = (x * b1) - (y * a1);
    if (block > 0 && (t + 1) % block == 0 && !(lv1 < -1.0e-8f || lv1 > 1.0e-8f)) lv1 = 0.0f;
    if (stages) stages[t] = y;
    /* Compressor<float>::processSample */
    const float a = fabsf(y);
    const float cte = (a > yold) ? cte_at : cte_rl;
    const float env = a + cte * (yold - a);
    yold = env;
    const float g = (env < thr) ? 1.0f : powf(env * thr_inv, ratio_inv - 1.0f);
    const float c = g * y;
    if (stages) stages[n + t] = c;
    /* Reverb::processMono */
    const float input = c * gain;
    float o = 0.0f;
    for (int j = 0; j < 8; ++j) {
      delay_line* d = &comb[j];
      const float output = d->buf[d->idx];
      d->last = (output * (1.0f - damp)) + (d->last * damp);
      UNDENORMALISE(d->last);
      float temp = input + (d->last * feedback);
      UNDENORMALISE(temp);
      d->buf[d->idx] = temp;
      d->idx = (d->idx + 1) % d->size;
      o += output;
    }
    for (int j = 0; j < 4; ++j) {
      delay_line* d = &ap[j];
      const float buffered = d->buf[d->idx];
      float temp = o + (buffered * 0.5f);
      UNDENORMALISE(temp);
      d->buf[d->idx] = temp;
      d->idx = (d->idx + 1) % d->size;
      o = buffered - o;
    }
    const float r = o * wet1 + c * dry;
    if (stages) stages[2 * n + t] = r;
    /* writeFromFloatArrays + 16-bit WAV writer */
    const double samp = (double)r;
    int32_t i32;
    if (samp <= -1.0) i32 = INT_MIN;
    else if (samp >= 1.0) i32 = INT_MAX;
    else i32 = (int32_t)nearbyint((double)INT_MAX * samp);
    out[t] = (int16_t)(i32 >> 16);
  }
  for (int j = 0; j < 8; ++j) free(comb[j].buf);
  for (int j = 0; j < 4; ++j) free(ap[j].buf);
  return 0;
}
