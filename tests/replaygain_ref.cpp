/* replaygain_ref.cpp -- ReplayGain analysis as lamejs runs it with gfp.findReplayGain = true: a statement-by-statement
 * restatement of src/js/GainAnalysis.js and src/js/ReplayGain.js (the buffers are Float32, the locals and sums double),
 * with the Java meaning where the JavaScript cannot run (`cursamples / 8` is an integer division, GainAnalysis.java).
 * Test infrastructure only: tests/replaygain_ref.py compiles it into a temporary directory and drives it with the pieces
 * lame_encode_buffer_sample hands to AnalyzeSamples (the n_out samples fill_buffer writes at mf_size).  Math.log10 is
 * fdlibm's (oracle/js_math.h), as on the device.
 *
 * Every completed RMS window is recorded: the bits of lsum and rsum and the histogram index it adds to A. */
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../oracle/js_math.h"

namespace {

const double STEPS_per_dB = 100., MAX_dB = 120., PINK_REF = 64.82, RMS_PERCENTILE = 0.95;
const int GAIN_NOT_ENOUGH_SAMPLES = -24601, MAX_ORDER = 10, MAX_SAMP_FREQ = 48000;
const int MAX_SAMPLES_PER_WINDOW = MAX_SAMP_FREQ * 1 / 20 + 1;
const int HIST = (int)(STEPS_per_dB * MAX_dB);

const double ABYule[9][21] = {
    {0.03857599435200, -3.84664617118067, -0.02160367184185, 7.81501653005538, -0.00123395316851, -11.34170355132042,
     -0.00009291677959, 13.05504219327545, -0.01655260341619, -12.28759895145294, 0.02161526843274, 9.48293806319790,
     -0.02074045215285, -5.87257861775999, 0.00594298065125, 2.75465861874613, 0.00306428023191, -0.86984376593551,
     0.00012025322027, 0.13919314567432, 0.00288463683916},
    {0.05418656406430, -3.47845948550071, -0.02911007808948, 6.36317777566148, -0.00848709379851, -8.54751527471874,
     -0.00851165645469, 9.47693607801280, -0.00834990904936, -8.81498681370155, 0.02245293253339, 6.85401540936998,
     -0.02596338512915, -4.39470996079559, 0.01624864962975, 2.19611684890774, -0.00240879051584, -0.75104302451432,
     0.00674613682247, 0.13149317958808, -0.00187763777362},
    {0.15457299681924, -2.37898834973084, -0.09331049056315, 2.84868151156327, -0.06247880153653, -2.64577170229825,
     0.02163541888798, 2.23697657451713, -0.05588393329856, -1.67148153367602, 0.04781476674921, 1.00595954808547,
     0.00222312597743, -0.45953458054983, 0.03174092540049, 0.16378164858596, -0.01390589421898, -0.05032077717131,
     0.00651420667831, 0.02347897407020, -0.00881362733839},
    {0.30296907319327, -1.61273165137247, -0.22613988682123, 1.07977492259970, -0.08587323730772, -0.25656257754070,
     0.03282930172664, -0.16276719120440, -0.00915702933434, -0.22638893773906, -0.02364141202522, 0.39120800788284,
     -0.00584456039913, -0.22138138954925, 0.06276101321749, 0.04500235387352, -0.00000828086748, 0.02005851806501,
     0.00205861885564, 0.00302439095741, -0.02950134983287},
    {0.33642304856132, -1.49858979367799, -0.25572241425570, 0.87350271418188, -0.11828570177555, 0.12205022308084,
     0.11921148675203, -0.80774944671438, -0.07834489609479, 0.47854794562326, -0.00469977914380, -0.12453458140019,
     -0.00589500224440, -0.04067510197014, 0.05724228140351, 0.08333755284107, 0.00832043980773, -0.04237348025746,
     -0.01635381384540, 0.02977207319925, -0.01760176568150},
    {0.44915256608450, -0.62820619233671, -0.14351757464547, 0.29661783706366, -0.22784394429749, -0.37256372942400,
     -0.01419140100551, 0.00213767857124, 0.04078262797139, -0.42029820170918, -0.12398163381748, 0.22199650564824,
     0.04097565135648, 0.00613424350682, 0.10478503600251, 0.06747620744683, -0.01863887810927, 0.05784820375801,
     -0.03193428438915, 0.03222754072173, 0.00541907748707},
    {0.56619470757641, -1.04800335126349, -0.75464456939302, 0.29156311971249, 0.16242137742230, -0.26806001042947,
     0.16744243493672, 0.00819999645858, -0.18901604199609, 0.45054734505008, 0.30931782841830, -0.33032403314006,
     -0.27562961986224, 0.06739368333110, 0.00647310677246, -0.04784254229033, 0.08647503780351, 0.01639907836189,
     -0.03788984554840, 0.01807364323573, -0.00588215443421},
    {0.58100494960553, -0.51035327095184, -0.53174909058578, -0.31863563325245, -0.14289799034253, -0.20256413484477,
     0.17520704835522, 0.14728154134330, 0.02377945217615, 0.38952639978999, 0.15558449135573, -0.23313271880868,
     -0.25344790059353, -0.05246019024463, 0.01628462406333, -0.02505961724053, 0.06920467763959, 0.02442357316099,
     -0.03721611395801, 0.01818801111503, -0.00749618797172},
    {0.53648789255105, -0.25049871956020, -0.42163034350696, -0.43193942311114, -0.00275953611929, -0.03424681017675,
     0.04267842219415, -0.04678328784242, -0.10214864179676, 0.26408300200955, 0.14590772289388, 0.15113130533216,
     -0.02459864859345, -0.17556493366449, -0.11202315195388, -0.18823009262115, -0.04060034127000, 0.05477720428674,
     0.04788665548180, 0.04704409688120, -0.02217936801134}};

const double ABButter[9][5] = {
    {0.98621192462708, -1.97223372919527, -1.97242384925416, 0.97261396931306, 0.98621192462708},
    {0.98500175787242, -1.96977855582618, -1.97000351574484, 0.97022847566350, 0.98500175787242},
    {0.97938932735214, -1.95835380975398, -1.95877865470428, 0.95920349965459, 0.97938932735214},
    {0.97531843204928, -1.95002759149878, -1.95063686409857, 0.95124613669835, 0.97531843204928},
    {0.97316523498161, -1.94561023566527, -1.94633046996323, 0.94705070426118, 0.97316523498161},
    {0.96454515552826, -1.92783286977036, -1.92909031105652, 0.93034775234268, 0.96454515552826},
    {0.96009142950541, -1.91858953033784, -1.92018285901082, 0.92177618768381, 0.96009142950541},
    {0.95856916599601, -1.91542108074780, -1.91713833199203, 0.91885558323625, 0.95856916599601},
    {0.94597685600279, -1.88903307939452, -1.89195371200558, 0.89487434461664, 0.94597685600279}};

struct ReplayGain {                     /* ReplayGain.js */
  float linprebuf[MAX_ORDER * 2], lstepbuf[MAX_SAMPLES_PER_WINDOW + MAX_ORDER], loutbuf[MAX_SAMPLES_PER_WINDOW + MAX_ORDER];
  float rinprebuf[MAX_ORDER * 2], rstepbuf[MAX_SAMPLES_PER_WINDOW + MAX_ORDER], routbuf[MAX_SAMPLES_PER_WINDOW + MAX_ORDER];
  int linpre, lstep, lout, rinpre, rstep, rout;
  int sampleWindow, totsamp;
  double lsum, rsum;
  int reqindex;
  int A[HIST], B[HIST];
  std::vector<uint64_t> trace;          /* per window: lsum bits, rsum bits, index */
};

void filterYule(const float* input, int inputPos, float* output, int outputPos, int nSamples, const double* kernel) {
  while ((nSamples--) != 0) {
    output[outputPos] = (float)(1e-10 + input[inputPos + 0] * kernel[0] - output[outputPos - 1] * kernel[1] +
                                input[inputPos - 1] * kernel[2] - output[outputPos - 2] * kernel[3] +
                                input[inputPos - 2] * kernel[4] - output[outputPos - 3] * kernel[5] +
                                input[inputPos - 3] * kernel[6] - output[outputPos - 4] * kernel[7] +
                                input[inputPos - 4] * kernel[8] - output[outputPos - 5] * kernel[9] +
                                input[inputPos - 5] * kernel[10] - output[outputPos - 6] * kernel[11] +
                                input[inputPos - 6] * kernel[12] - output[outputPos - 7] * kernel[13] +
                                input[inputPos - 7] * kernel[14] - output[outputPos - 8] * kernel[15] +
                                input[inputPos - 8] * kernel[16] - output[outputPos - 9] * kernel[17] +
                                input[inputPos - 9] * kernel[18] - output[outputPos - 10] * kernel[19] +
                                input[inputPos - 10] * kernel[20]);
    ++outputPos;
    ++inputPos;
  }
}

void filterButter(const float* input, int inputPos, float* output, int outputPos, int nSamples, const double* kernel) {
  while ((nSamples--) != 0) {
    output[outputPos] = (float)(input[inputPos + 0] * kernel[0] - output[outputPos - 1] * kernel[1] +
                                input[inputPos - 1] * kernel[2] - output[outputPos - 2] * kernel[3] +
                                input[inputPos - 2] * kernel[4]);
    ++outputPos;
    ++inputPos;
  }
}

int ResetSampleFrequency(ReplayGain* g, int samplefreq) {
  for (int i = 0; i < MAX_ORDER; i++)
    g->linprebuf[i] = g->lstepbuf[i] = g->loutbuf[i] = g->rinprebuf[i] = g->rstepbuf[i] = g->routbuf[i] = 0.f;
  switch (samplefreq) {
    case 48000: g->reqindex = 0; break;
    case 44100: g->reqindex = 1; break;
    case 32000: g->reqindex = 2; break;
    case 24000: g->reqindex = 3; break;
    case 22050: g->reqindex = 4; break;
    case 16000: g->reqindex = 5; break;
    case 12000: g->reqindex = 6; break;
    case 11025: g->reqindex = 7; break;
    case 8000: g->reqindex = 8; break;
    default: return 0;
  }
  g->sampleWindow = (samplefreq * 1 + 20 - 1) / 20;
  g->lsum = 0.;
  g->rsum = 0.;
  g->totsamp = 0;
  memset(g->A, 0, sizeof g->A);             /* `Arrays.ill(rgData.A, 0)`: Arrays.fill */
  return 1;
}

inline double fsqr(double d) { return d * d; }

double analyzeResult(const int* Array, int len) {
  long long elems = 0;
  int i;
  for (i = 0; i < len; i++) elems += Array[i];
  if (elems == 0) return GAIN_NOT_ENOUGH_SAMPLES;
  long long upper = (long long)ceil((double)elems * (1. - RMS_PERCENTILE));
  for (i = len; i-- > 0;) {
    if ((upper -= Array[i]) <= 0) break;
  }
  return (PINK_REF - i / STEPS_per_dB);
}

}  // namespace

extern "C" {

void* rg_create(int samplefreq) {
  ReplayGain* g = new ReplayGain();
  if (!ResetSampleFrequency(g, samplefreq)) { delete g; return nullptr; }
  g->linpre = g->rinpre = g->lstep = g->rstep = g->lout = g->rout = MAX_ORDER;   /* InitGainAnalysis */
  memset(g->B, 0, sizeof g->B);
  return g;
}

void rg_destroy(void* h) { delete (ReplayGain*)h; }

int rg_sample_window(void* h) { return ((ReplayGain*)h)->sampleWindow; }

/* AnalyzeSamples(rgData, left, 0, right, 0, num_samples, num_channels) */
int rg_analyze(void* h, const float* left_samples, const float* right_samples, int num_samples, int num_channels) {
  ReplayGain* g = (ReplayGain*)h;
  const float* curleftBase;
  const float* currightBase;
  int curleft, curright, batchsamples, cursamples, cursamplepos;
  if (num_samples == 0) return 1;
  cursamplepos = 0;
  batchsamples = num_samples;
  switch (num_channels) {
    case 1: right_samples = left_samples; break;
    case 2: break;
    default: return 0;
  }
  if (num_samples < MAX_ORDER) {
    memcpy(g->linprebuf + MAX_ORDER, left_samples, sizeof(float) * num_samples);
    memcpy(g->rinprebuf + MAX_ORDER, right_samples, sizeof(float) * num_samples);
  } else {
    memcpy(g->linprebuf + MAX_ORDER, left_samples, sizeof(float) * MAX_ORDER);
    memcpy(g->rinprebuf + MAX_ORDER, right_samples, sizeof(float) * MAX_ORDER);
  }
  while (batchsamples > 0) {
    cursamples = batchsamples > g->sampleWindow - g->totsamp ? g->sampleWindow - g->totsamp : batchsamples;
    if (cursamplepos < MAX_ORDER) {
      curleft = g->linpre + cursamplepos;
      curleftBase = g->linprebuf;
      curright = g->rinpre + cursamplepos;
      currightBase = g->rinprebuf;
      if (cursamples > MAX_ORDER - cursamplepos) cursamples = MAX_ORDER - cursamplepos;
    } else {
      curleft = cursamplepos;
      curleftBase = left_samples;
      curright = cursamplepos;
      currightBase = right_samples;
    }
    filterYule(curleftBase, curleft, g->lstepbuf, g->lstep + g->totsamp, cursamples, ABYule[g->reqindex]);
    filterYule(currightBase, curright, g->rstepbuf, g->rstep + g->totsamp, cursamples, ABYule[g->reqindex]);
    filterButter(g->lstepbuf, g->lstep + g->totsamp, g->loutbuf, g->lout + g->totsamp, cursamples, ABButter[g->reqindex]);
    filterButter(g->rstepbuf, g->rstep + g->totsamp, g->routbuf, g->rout + g->totsamp, cursamples, ABButter[g->reqindex]);

    curleft = g->lout + g->totsamp;
    const float* lo = g->loutbuf;
    curright = g->rout + g->totsamp;
    const float* ro = g->routbuf;
    int i = cursamples % 8;
    while ((i--) != 0) {
      g->lsum += fsqr(lo[curleft++]);
      g->rsum += fsqr(ro[curright++]);
    }
    i = cursamples / 8;                       /* an integer division in Java (JavaScript: a fraction, and no end) */
    while ((i--) != 0) {
      g->lsum += fsqr(lo[curleft + 0]) + fsqr(lo[curleft + 1]) + fsqr(lo[curleft + 2]) + fsqr(lo[curleft + 3]) +
                 fsqr(lo[curleft + 4]) + fsqr(lo[curleft + 5]) + fsqr(lo[curleft + 6]) + fsqr(lo[curleft + 7]);
      curleft += 8;
      g->rsum += fsqr(ro[curright + 0]) + fsqr(ro[curright + 1]) + fsqr(ro[curright + 2]) + fsqr(ro[curright + 3]) +
                 fsqr(ro[curright + 4]) + fsqr(ro[curright + 5]) + fsqr(ro[curright + 6]) + fsqr(ro[curright + 7]);
      curright += 8;
    }
    batchsamples -= cursamples;
    cursamplepos += cursamples;
    g->totsamp += cursamples;
    if (g->totsamp == g->sampleWindow) {
      const double val = STEPS_per_dB * 10. * js_log10((g->lsum + g->rsum) / g->totsamp * 0.5 + 1.e-37);
      int ival = (val <= 0) ? 0 : (int)val;
      if (ival >= HIST) ival = HIST - 1;
      g->A[ival]++;
      uint64_t lb, rb;
      memcpy(&lb, &g->lsum, 8);
      memcpy(&rb, &g->rsum, 8);
      g->trace.push_back(lb); g->trace.push_back(rb); g->trace.push_back((uint64_t)ival);
      g->lsum = g->rsum = 0.;
      memmove(g->loutbuf, g->loutbuf + g->totsamp, sizeof(float) * MAX_ORDER);
      memmove(g->routbuf, g->routbuf + g->totsamp, sizeof(float) * MAX_ORDER);
      memmove(g->lstepbuf, g->lstepbuf + g->totsamp, sizeof(float) * MAX_ORDER);
      memmove(g->rstepbuf, g->rstepbuf + g->totsamp, sizeof(float) * MAX_ORDER);
      g->totsamp = 0;
    }
    if (g->totsamp > g->sampleWindow) return 0;
  }
  if (num_samples < MAX_ORDER) {
    memmove(g->linprebuf, g->linprebuf + num_samples, sizeof(float) * (MAX_ORDER - num_samples));
    memmove(g->rinprebuf, g->rinprebuf + num_samples, sizeof(float) * (MAX_ORDER - num_samples));
    memcpy(g->linprebuf + MAX_ORDER - num_samples, left_samples, sizeof(float) * num_samples);
    memcpy(g->rinprebuf + MAX_ORDER - num_samples, right_samples, sizeof(float) * num_samples);
  } else {
    memcpy(g->linprebuf, left_samples + num_samples - MAX_ORDER, sizeof(float) * MAX_ORDER);
    memcpy(g->rinprebuf, right_samples + num_samples - MAX_ORDER, sizeof(float) * MAX_ORDER);
  }
  return 1;
}

/* GetTitleGain: the title's gain; A moves into B and the filters restart from zero */
double rg_title_gain(void* h) {
  ReplayGain* g = (ReplayGain*)h;
  const double retval = analyzeResult(g->A, HIST);
  for (int i = 0; i < HIST; i++) { g->B[i] += g->A[i]; g->A[i] = 0; }
  for (int i = 0; i < MAX_ORDER; i++)
    g->linprebuf[i] = g->lstepbuf[i] = g->loutbuf[i] = g->rinprebuf[i] = g->rstepbuf[i] = g->routbuf[i] = 0.f;
  g->totsamp = 0;
  g->lsum = g->rsum = 0.;
  return retval;
}

/* GetAlbumGain (LAME gain_analysis.c): the same rule over B */
double rg_album_gain(void* h) { return analyzeResult(((ReplayGain*)h)->B, HIST); }

/* analyzeResult over a caller's histogram (HIST bins) */
double rg_analyze_result(const int* hist) { return analyzeResult(hist, HIST); }

/* the windows recorded so far (3 words each); copies min(n, count) of them into out when out != NULL */
long long rg_trace(void* h, uint64_t* out, long long n) {
  ReplayGain* g = (ReplayGain*)h;
  const long long k = (long long)g->trace.size() / 3;
  if (out) memcpy(out, g->trace.data(), sizeof(uint64_t) * 3 * (size_t)(n < k ? n : k));
  return k;
}

void rg_hist(void* h, int* a, int* b) {
  ReplayGain* g = (ReplayGain*)h;
  if (a) memcpy(a, g->A, sizeof g->A);
  if (b) memcpy(b, g->B, sizeof g->B);
}
}
