/* k_replaygain.cuh -- ReplayGain analysis (lamejs GainAnalysis.js with gfp.findReplayGain = true) on the device.
 *
 * lamejs runs every sample it puts into mfbuf through a 10th-order Yule-Walker IIR and a 2nd-order Butterworth, each
 * output rounded to Float32 and each sum done in double left to right, then sums the squares of the result per RMS window
 * (sampleWindow = ceil(rate / 20) samples) and adds each window's level to a 12000-bin histogram.  The filter is one long
 * recurrence per channel with about 20 dependent double adds per sample, and its rounding forbids any reordering.  It is
 * evaluated here by speculation and verification, like k_stream_scan:
 *   k_rg_pass1   a title's complete windows are cut into chunks of RG_CHUNK_WINDOWS windows; every (chunk, channel) runs
 *                from a guessed state (RG_GUESS) and records the state at each of its window ends and each window's sum;
 *   k_rg_repair  a chunk whose assumed start state differs (bitwise) from its predecessor's end state runs again from the
 *                true state, and stops at the first window end whose state equals the one it recorded before: from there
 *                on every value is the same.  A chunk that changed its end state makes another pass necessary;
 *   k_rg_check   ends the passes once one of them changed no end state.
 * The state at a window end is 12 Float32 values per channel (the last 10 Yule outputs and the last 2 Butterworth
 * outputs); the filters' inputs are the samples themselves and are read again.  The guess changes the speed only.
 *
 * A window's sum depends on how lamejs split the samples into AnalyzeSamples calls: each call ("piece") and each window
 * starts a new run of `n % 8` single adds followed by groups of eight, and a piece's first MAX_ORDER samples are a run of
 * their own.  The host passes each title's piece starts.
 * A launch analyses the samples [g0, g1) of a title that started at t0 (stream sample indices): a whole stream is [0, end),
 * a streaming handle continues from the state and partial window sums it carries (RgCarry) and keeps them for its next call;
 * chunk 0 starts from that carried state, which is exact, the later chunks at window starts.
 *   k_rg_hist    window -> histogram index (1000 log10(mean square / 2 + 1e-37), fdlibm's log10), integer atomics;
 *   k_rg_result  analyzeResult of a histogram (GainAnalysis.js:515-532); k_rg_album sums the histograms of a batch first.
 *
 * Included after every other kernel header, so that its __constant__ tables sit behind theirs.
 */
#ifndef MP3B200_K_REPLAYGAIN_CUH
#define MP3B200_K_REPLAYGAIN_CUH
#include "mp3_device.cuh"
#include "mp3_math.cuh"

#ifndef RG_CHUNK_WINDOWS
#define RG_CHUNK_WINDOWS 4              /* windows per speculated chunk (speed only) */
#endif
#ifndef RG_GUESS
#define RG_GUESS 0                      /* 0: a chunk starts from the zero state; 1: from a deliberately wrong state (tests) */
#endif
#ifndef RG_QUEUED_PASSES
#define RG_QUEUED_PASSES 4              /* repair passes queued without waiting for the host (more run if needed; speed only) */
#endif
#define RG_THREADS 64
#define RG_HIST 12000
#define RG_ORDER 10
#define RG_NOT_ENOUGH_SAMPLES (-24601)

__constant__ double c_rg_yule[9][21];
__constant__ double c_rg_butter[9][5];

/* GainAnalysis.js:154-237: the filters of the nine analysis rates (48000, 44100, 32000, 24000, 22050, 16000, 12000, 11025,
 * 8000 Hz), uploaded into c_rg_yule / c_rg_butter */
static const double RG_YULE[9][21] = {
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

static const double RG_BUTTER[9][5] = {
    {0.98621192462708, -1.97223372919527, -1.97242384925416, 0.97261396931306, 0.98621192462708},
    {0.98500175787242, -1.96977855582618, -1.97000351574484, 0.97022847566350, 0.98500175787242},
    {0.97938932735214, -1.95835380975398, -1.95877865470428, 0.95920349965459, 0.97938932735214},
    {0.97531843204928, -1.95002759149878, -1.95063686409857, 0.95124613669835, 0.97531843204928},
    {0.97316523498161, -1.94561023566527, -1.94633046996323, 0.94705070426118, 0.97316523498161},
    {0.96454515552826, -1.92783286977036, -1.92909031105652, 0.93034775234268, 0.96454515552826},
    {0.96009142950541, -1.91858953033784, -1.92018285901082, 0.92177618768381, 0.96009142950541},
    {0.95856916599601, -1.91542108074780, -1.91713833199203, 0.91885558323625, 0.95856916599601},
    {0.94597685600279, -1.88903307939452, -1.89195371200558, 0.89487434461664, 0.94597685600279}};

struct RgState { float y[RG_ORDER]; float z[2]; };      /* y[0] / z[0]: the newest output */
struct RgEnd { RgState st; double sum; };                /* a chunk's end: the state, and the partial window sum there */
struct RgCarry { RgState st[2]; double sum[2]; };        /* what a handle carries between launches, per channel */

struct RgTitle {
  const void* x[2];            /* channel rows: int16 (scaled like mfbuf) or Float32 (the resampler's output) */
  long long x_base, x_end;     /* samples [x_base, x_end) are x[c][j - x_base]; later ones (the flush's zeros) are 0 */
  const long long* piece;      /* starts of the pieces AnalyzeSamples saw in [g0, g1), ascending, piece[0] = g0 */
  int npieces;
  long long t0, g0, g1;        /* title start; the samples this launch analyses */
  int wa, nwin, win0;          /* window (of the title) g0 lies in; windows completed in [g0, g1); first row in the window arrays */
  int nchunks, chunk0;         /* chunks, first row in the chunk arrays */
  RgCarry* carry;              /* in: state and sums at g0; after k_rg_finish: at g1 (zero after a title end) */
  int* hist;                   /* histogram A of the title */
  int* hist_b;                 /* B (GetTitleGain adds A to it and clears A); NULL: leave A */
  int title_end;               /* GetTitleGain after g1 */
};

__device__ __forceinline__ float rg_x(const RgTitle& t, int c, long long j, bool f32, int scale_applied, double scale) {
  if (j < t.x_base || j >= t.x_end) return 0.f;
  const long long i = j - t.x_base;
  if (f32) return static_cast<const float*>(t.x[c])[i];
  double d = (double)static_cast<const int16_t*>(t.x[c])[i];
  if (scale_applied) d = (double)(float)(d * scale);
  return (float)d;
}

/* one sample through both filters (GainAnalysis.js filterYule / filterButter); returns the squared output */
__device__ __forceinline__ double rg_step(float xin, float (&xh)[RG_ORDER], float (&yh)[RG_ORDER], float (&zh)[2],
                                          const double (&K)[21], const double (&B)[5]) {
  double acc = 1e-10 + (double)xin * K[0];
#pragma unroll
  for (int k = 0; k < RG_ORDER; k++) {
    acc = acc - (double)yh[k] * K[2 * k + 1];
    acc = acc + (double)xh[k] * K[2 * k + 2];
  }
  const float y = (float)acc;
  const float z = (float)((double)y * B[0] - (double)zh[0] * B[1] + (double)yh[0] * B[2] - (double)zh[1] * B[3] + (double)yh[1] * B[4]);
#pragma unroll
  for (int k = RG_ORDER - 1; k > 0; k--) { xh[k] = xh[k - 1]; yh[k] = yh[k - 1]; }
  xh[0] = xin; yh[0] = y;
  zh[1] = zh[0]; zh[0] = z;
  return (double)z * (double)z;
}

__device__ __forceinline__ bool rg_same(const RgState& a, const RgState& b) {
  bool eq = true;
#pragma unroll
  for (int k = 0; k < RG_ORDER; k++) eq &= __float_as_uint(a.y[k]) == __float_as_uint(b.y[k]);
  eq &= __float_as_uint(a.z[0]) == __float_as_uint(b.z[0]) && __float_as_uint(a.z[1]) == __float_as_uint(b.z[1]);
  return eq;
}

__device__ __forceinline__ RgState rg_guess() {
  RgState s;
#pragma unroll
  for (int k = 0; k < RG_ORDER; k++) s.y[k] = RG_GUESS ? 1000.f * (k + 1) : 0.f;
  s.z[0] = RG_GUESS ? -500.f : 0.f; s.z[1] = RG_GUESS ? 250.f : 0.f;
  return s;
}

/* the samples chunk k of title t covers: windows wa + k CW .. wa + (k + 1) CW - 1, clipped to [g0, g1) */
__device__ __forceinline__ void rg_chunk_span(const RgTitle& t, int W, int k, long long& j0, long long& j1) {
  j0 = t.t0 + (long long)(t.wa + k * RG_CHUNK_WINDOWS) * W;
  j1 = j0 + (long long)RG_CHUNK_WINDOWS * W;
  if (j0 < t.g0) j0 = t.g0;
  if (j1 > t.g1) j1 = t.g1;
}

/* Runs samples [j0, j1) of title t, channel c, from state `st` and partial window sum `lsum`.  Writes the sum (mono: both
 * slots) and end state of every window completed on the way; with Repair, stops at the first window whose end state equals
 * the recorded one and returns true.  Otherwise `st` / `lsum` are the state and partial sum at j1. */
template <bool Repair>
__device__ bool rg_run(const RgTitle& t, int c, int nch, int W, int req, bool f32, int scale_applied, double scale, long long j0,
                       long long j1, RgState& st, double& lsum, double* __restrict__ win_sum, RgState* __restrict__ win_state) {
  double K[21], B[5];
#pragma unroll
  for (int k = 0; k < 21; k++) K[k] = c_rg_yule[req][k];
#pragma unroll
  for (int k = 0; k < 5; k++) B[k] = c_rg_butter[req][k];
  float xh[RG_ORDER], yh[RG_ORDER], zh[2];
#pragma unroll
  for (int k = 0; k < RG_ORDER; k++) {   /* the title's input starts with zeros (the prebuffer InitGainAnalysis / GetTitleGain clear) */
    const long long jk = j0 - 1 - k;
    xh[k] = jk < t.t0 ? 0.f : rg_x(t, c, jk, f32, scale_applied, scale);
    yh[k] = st.y[k];
  }
  zh[0] = st.z[0]; zh[1] = st.z[1];
  int lo = 0, hi = t.npieces;                       /* pi = first piece starting after j0 */
  while (lo < hi) { const int m = (lo + hi) >> 1; if (t.piece[m] <= j0) lo = m + 1; else hi = m; }
  int pi = lo;
  long long j = j0;
  double sum = lsum;
  while (j < j1) {
    const long long we = t.t0 + ((j - t.t0) / W + 1) * W;       /* the end of the window j lies in */
    const long long stop = we < j1 ? we : j1;
    while (j < stop) {
      while (pi < t.npieces && t.piece[pi] <= j) pi++;
      long long e = pi < t.npieces ? t.piece[pi] : stop;
      if (pi > 0) { const long long q = t.piece[pi - 1] + RG_ORDER; if (q > j && q < e) e = q; }
      if (e > stop) e = stop;
      const int n = (int)(e - j), r = n % 8;
      for (int i = 0; i < r; i++, j++) sum += rg_step(rg_x(t, c, j, f32, scale_applied, scale), xh, yh, zh, K, B);
      for (int g = 0; g < n / 8; g++) {
        double grp = rg_step(rg_x(t, c, j, f32, scale_applied, scale), xh, yh, zh, K, B);
        j++;
#pragma unroll
        for (int i = 1; i < 8; i++, j++) grp = grp + rg_step(rg_x(t, c, j, f32, scale_applied, scale), xh, yh, zh, K, B);
        sum += grp;
      }
    }
    RgState ns;
#pragma unroll
    for (int k = 0; k < RG_ORDER; k++) ns.y[k] = yh[k];
    ns.z[0] = zh[0]; ns.z[1] = zh[1];
    if (j == we) {                                              /* a window completed */
      const long long row = (long long)t.win0 + ((we - t.t0) / W - 1 - t.wa);
      win_sum[row * 2 + c] = sum;
      if (nch == 1) win_sum[row * 2 + 1] = sum;
      RgState& rec = win_state[row * nch + c];
      if (Repair && rg_same(ns, rec)) return true;
      rec = ns;
      sum = 0.0;
    }
    st = ns;
  }
  lsum = sum;
  return false;
}

struct RgParams {
  const RgTitle* titles;
  int nch, W, req, f32, scale_applied;
  double scale;
  double* win_sum;             /* [windows][2] lsum, rsum */
  RgState* win_state;          /* [windows][nch] */
  RgState* chunk_start;        /* [chunks][nch] the state each chunk was last run from */
  RgEnd* end_in;               /* [chunks][nch] end states: read by a pass ... */
  RgEnd* end_out;              /* ... written by it */
  int* pass_changed;           /* [passes] chunks whose end state a pass changed */
  int* done;                   /* 1 once a pass changed nothing */
  int* reruns;                 /* chunks run again, over all passes */
};

/* grid (ceil(max chunks * nch / RG_THREADS), titles); thread = (chunk, channel).  Chunk 0 starts from the carried state, the
 * others from the guess. */
__global__ void __launch_bounds__(RG_THREADS) k_rg_pass1(RgParams p) {
  const RgTitle t = p.titles[blockIdx.y];
  const int i = blockIdx.x * RG_THREADS + threadIdx.x;
  if (i >= t.nchunks * p.nch) return;
  const int k = i / p.nch, c = i % p.nch;
  long long j0, j1;
  rg_chunk_span(t, p.W, k, j0, j1);
  RgState st = k == 0 ? t.carry->st[c] : rg_guess();
  double sum = k == 0 ? t.carry->sum[c] : 0.0;
  const long long row = ((long long)t.chunk0 + k) * p.nch + c;
  p.chunk_start[row] = st;
  rg_run<false>(t, c, p.nch, p.W, p.req, p.f32, p.scale_applied, p.scale, j0, j1, st, sum, p.win_sum, p.win_state);
  p.end_in[row] = RgEnd{st, sum};
}

/* one repair pass, thread = (chunk, channel) as in k_rg_pass1.  The pass index is `pass`, or with At what `at` points to,
 * read where it is used so that it holds no register through the run. */
template <bool At>
__device__ __forceinline__ void rg_repair_pass(const RgParams& p, int pass, const int* at) {
  if (*p.done) return;
  const RgTitle t = p.titles[blockIdx.y];
  const int i = blockIdx.x * RG_THREADS + threadIdx.x;
  if (i >= t.nchunks * p.nch) return;
  const int k = i / p.nch, c = i % p.nch;
  const long long row = ((long long)t.chunk0 + k) * p.nch + c;
  const RgState truth = k == 0 ? t.carry->st[c] : p.end_in[row - p.nch].st;
  if (rg_same(truth, p.chunk_start[row])) { p.end_out[row] = p.end_in[row]; return; }
  p.chunk_start[row] = truth;
  atomicAdd(p.reruns, 1);
  long long j0, j1;
  rg_chunk_span(t, p.W, k, j0, j1);
  RgState st = truth;
  double sum = k == 0 ? t.carry->sum[c] : 0.0;
  const bool merged = rg_run<true>(t, c, p.nch, p.W, p.req, p.f32, p.scale_applied, p.scale, j0, j1, st, sum, p.win_sum, p.win_state);
  if (merged) { p.end_out[row] = p.end_in[row]; return; }
  p.end_out[row] = RgEnd{st, sum};
  if (!rg_same(st, p.end_in[row].st) || __double_as_longlong(sum) != __double_as_longlong(p.end_in[row].sum))
    atomicAdd(p.pass_changed + (At ? *at : pass), 1);
}

/* after pass `pass`: done when it changed no end state; otherwise its end states become the next pass's input */
__device__ __forceinline__ void rg_check_pass(const RgParams& p, int pass, long long rows) {
  if (*p.done) return;
  const bool stop = p.pass_changed[pass] == 0;
  for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (long long)gridDim.x * blockDim.x)
    p.end_in[r] = p.end_out[r];
  if (stop && blockIdx.x == 0 && threadIdx.x == 0) *p.done = 1;
}

__global__ void __launch_bounds__(RG_THREADS) k_rg_repair(RgParams p, int pass) { rg_repair_pass<false>(p, pass, nullptr); }
__global__ void k_rg_check(RgParams p, int pass, long long rows) { rg_check_pass(p, pass, rows); }

/* ---- the repair loop on the device (an encode session's tagged calls: no host round trip per pass) ----
 * A CUDA graph whose conditional WHILE node has one pass as its body: k_rg_repair_at and k_rg_check_at, which are k_rg_repair
 * and k_rg_check taking the pass index from device memory, then k_rg_loop_cond.  loop[0] is that index (the host sets it to
 * RG_QUEUED_PASSES, the passes queued ahead of the graph); k_rg_report leaves the counts of the call in loop[1 .. 2]. */
__global__ void __launch_bounds__(RG_THREADS) k_rg_repair_at(RgParams p, const int* loop) { rg_repair_pass<true>(p, 0, loop); }
__global__ void k_rg_check_at(RgParams p, const int* __restrict__ loop, long long rows) { rg_check_pass(p, loop[0], rows); }

/* one thread, after each pass of the body: counts it and lets the body run again unless a pass has changed nothing.  With
 * max_passes run and still no such pass (the bound of the host loop, rg_finish, which cannot be reached) it ends the loop
 * with *fault = RG_FAULT. */
#define RG_FAULT 2
__global__ void k_rg_loop_cond(cudaGraphConditionalHandle handle, int* __restrict__ loop, int* __restrict__ done, int max_passes,
                               int* __restrict__ fault) {
  const int passes = loop[0] + 1;
  loop[0] = passes;
  bool more = *done == 0;
  if (more && passes >= max_passes) { *done = 1; *fault = RG_FAULT; more = false; }
  cudaGraphSetConditional(handle, more ? 1u : 0u);
}

/* one thread, after the loop: loop[1] = the passes the analysis needed, counted like rg_finish counts them -- up to and
 * including the first of the loop[0] passes run that changed nothing (later ones returned at once); loop[2] = chunks run again */
__global__ void k_rg_report(int* __restrict__ loop, const int* __restrict__ pass_changed, const int* __restrict__ reruns) {
  int used = 0;
  while (used < loop[0] && pass_changed[used] != 0) used++;
  loop[1] = used + 1;
  loop[2] = *reruns;
}

/* grid (ceil(max windows / 256), titles): histogram index of every completed window (GainAnalysis.js:466-475) */
__global__ void k_rg_hist(const RgTitle* __restrict__ titles, int W, const double* __restrict__ win_sum, int* __restrict__ win_idx) {
  const RgTitle t = titles[blockIdx.y];
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= t.nwin) return;
  const long long row = (long long)t.win0 + w;
  const double val = 100. * 10. * m3_log10((win_sum[2 * row] + win_sum[2 * row + 1]) / W * 0.5 + 1.e-37);
  int ival = (val <= 0) ? 0 : (int)val;
  if (ival >= RG_HIST) ival = RG_HIST - 1;
  win_idx[row] = ival;
  atomicAdd(t.hist + ival, 1);
}

/* album histogram: bin-wise sum over the titles' histograms A */
__global__ void k_rg_album(const RgTitle* __restrict__ titles, int ntitles, int* __restrict__ album) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= RG_HIST) return;
  int s = 0;
  for (int t = 0; t < ntitles; t++) s += titles[t].hist[b];
  album[b] = s;
}

/* analyzeResult (GainAnalysis.js:515-532): the largest i whose bins i .. end hold ceil(elems * 0.05) windows */
__host__ __device__ inline double rg_analyze_result(const int* A) {
  long long elems = 0;
  for (int i = 0; i < RG_HIST; i++) elems += A[i];
  if (elems == 0) return RG_NOT_ENOUGH_SAMPLES;
  long long upper = (long long)ceil((double)elems * (1. - 0.95));
  int i;
  for (i = RG_HIST; i-- > 0;)
    if ((upper -= A[i]) <= 0) break;
  return 64.82 - i / 100.;
}

/* one block of 256 per histogram (hists[b]; a title that does not end this launch is skipped): analyzeResult */
__global__ void __launch_bounds__(256) k_rg_result(const RgTitle* __restrict__ titles, int ntitles, const int* __restrict__ album,
                                                   double* __restrict__ gain) {
  const bool is_album = (int)blockIdx.x == ntitles;
  if (!is_album && !titles[blockIdx.x].title_end) return;
  const int* A = is_album ? album : titles[blockIdx.x].hist;
  __shared__ long long part[256];
  __shared__ long long suffix[257];
  constexpr int PER = (RG_HIST + 255) / 256;
  const int lo = threadIdx.x * PER, hi = min(lo + PER, RG_HIST);
  long long s = 0;
  for (int i = lo; i < hi; i++) s += A[i];
  part[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    suffix[256] = 0;
    for (int q = 255; q >= 0; q--) suffix[q] = suffix[q + 1] + part[q];
  }
  __syncthreads();
  const long long elems = suffix[0];
  if (elems == 0) { if (threadIdx.x == 0) gain[blockIdx.x] = RG_NOT_ENOUGH_SAMPLES; return; }
  const long long upper = (long long)ceil((double)elems * (1. - 0.95));
  if (suffix[threadIdx.x + 1] < upper && suffix[threadIdx.x] >= upper) {
    long long acc = suffix[threadIdx.x + 1];
    int i = hi - 1;
    for (; i >= lo; i--) { acc += A[i]; if (acc >= upper) break; }
    gain[blockIdx.x] = 64.82 - i / 100.;
  }
}

/* grid (titles): the carry a title keeps for its next launch -- the last chunk's end, or zeros after GetTitleGain, which also
 * adds A to B and clears A (GainAnalysis.js:534-548) */
__global__ void __launch_bounds__(256) k_rg_finish(const RgTitle* __restrict__ titles, const RgEnd* __restrict__ end, int nch) {
  const RgTitle t = titles[blockIdx.x];
  if (t.title_end) {
    if (t.hist_b)
      for (int b = threadIdx.x; b < RG_HIST; b += blockDim.x) { t.hist_b[b] += t.hist[b]; t.hist[b] = 0; }
    if (threadIdx.x < 2) {
      RgState z;
      for (int k = 0; k < RG_ORDER; k++) z.y[k] = 0.f;
      z.z[0] = z.z[1] = 0.f;
      t.carry->st[threadIdx.x] = z;
      t.carry->sum[threadIdx.x] = 0.0;
    }
  } else if (t.nchunks > 0 && threadIdx.x < 2) {
    const int c = nch == 1 ? 0 : threadIdx.x;
    const RgEnd e = end[((long long)t.chunk0 + t.nchunks - 1) * nch + c];
    t.carry->st[threadIdx.x] = e.st;
    t.carry->sum[threadIdx.x] = e.sum;
  }
}

#endif
