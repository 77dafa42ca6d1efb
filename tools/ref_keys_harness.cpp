// tools/ref_keys_harness.cpp — the reference's own remote loop: ESPFlix::loop() and key_event() (espflix.cpp:886-1040) run as they are,
// compiled from the UNMODIFIED espflix.cpp, for tools/make_keys_golden.py. TEST INFRASTRUCTURE ONLY.
//
// As tools/ref_nav_harness.cpp: espflix.cpp is included whole under `#define class struct` with every standard header first, and the
// symbols it references are stubbed. loop() itself runs: get_nec() hands it the script's NEC codes one iteration at a time and throws
// after the last one, which is how the harness leaves loop(). The Wi-Fi GUI passes keys through (_wifi_state and wifi_state() are
// CONNECTED). The decoder is instant: clear_events(DECODER_RUN) pauses it at once (get_events() reports DECODER_PAUSED whenever RUN is
// clear), and a Streamer::read() of 0 bytes ends the stream and pauses it, as MpegDecoder::pause() does on a 0-byte Buffer
// (player.cpp:1345-1346). A poster reads 0 bytes at once, so load_poster() returns; a title's file reads 0 bytes only in the iteration
// a script step marks as the end of the title.
//
// A script step is (nec, ended, pts): when ended, one idle iteration whose read ends the title (loop() sets _pending = DONE); then the
// key iteration with get_nec() = nec; then one idle iteration, so that a pending action resolves. get_pts() = pts throughout the step.
// Per step the harness reports what tools/ref_nav_harness.cpp reports, plus _video_composite_blend and _last_seconds. Both are set to
// a sentinel when the step starts, so the report says whether the step wrote them. update_progress(), which the idle iterations run,
// redraws the clock; the clock is the present calls' business (ef_present_clock), so its write of _last_seconds is undone: the value
// before it is captured where the idle iteration reaches the decoder (pop_empty() of a title's file) or sleeps (usleep), and put back
// when the next iteration starts.
#include <math.h>
#include <pthread.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

#include <algorithm>
#include <condition_variable>
#include <deque>
#include <functional>
#include <list>
#include <map>
#include <mutex>
#include <queue>
#include <string>
#include <thread>
#include <vector>

static void efref_idle();
#define usleep(us) efref_idle()
#define class struct
#include "espflix.cpp"
#undef class
#undef usleep

static const int kSentinel = 0x5EED;
static int64_t g_pts = -1;
extern "C" { uint8_t efref_composite_area[VIDEO_COMPOSITE_HEIGHT * VIDEO_COMPOSITE_WIDTH + 4096]; }
extern uint8_t _video_composite[VIDEO_COMPOSITE_HEIGHT * VIDEO_COMPOSITE_WIDTH] __attribute__((alias("efref_composite_area")));
int _video_composite_blend;
int _video_composite_progress;

static std::string g_url, g_cur_url;                         // the file asked for in this step; the file being read
static uint32_t g_offset = 0;
static int g_mode = -1;
static int g_writes = 0;
static bool g_run = false, g_end = false;
static std::map<std::string, int64_t> g_nv;
static std::vector<std::vector<uint8_t>> g_idx;              // every title's video.idx image
static Buffer g_buffer;
static ESPFlix* g_player = nullptr;
static bool g_captured = false;
static int64_t g_capture = 0;

struct Done {};                                              // thrown by get_nec() after the last iteration

static bool poster_open() { return g_cur_url.find("poster.ts") != std::string::npos; }
static void efref_idle() { g_captured = true; g_capture = g_player->_last_seconds; }

void Frame::init() {}
uint8_t* Frame::get_y(int) { return efref_composite_area; }
void Frame::erase() {}
MpegDecoder::MpegDecoder(Frame*, Frame*) {}
void MpegDecoder::flush_picture(int mode) { g_mode = mode; }
int64_t MpegDecoder::get_pts() { return g_pts; }
Buffer* MpegDecoder::pop_empty()
{
    if (!poster_open()) efref_idle();                        // loop()'s decode_next(), not load_poster()'s
    return &g_buffer;
}
void MpegDecoder::push_full(Buffer*) {}
void MpegDecoder::reset() {}
void MpegDecoder::run() {}
int Streamer::get(const char* url, uint32_t offset, uint32_t) { g_url = g_cur_url = url; g_offset = offset; return 0; }
void Streamer::get_rom(const uint8_t*, int) {}
static int title_of(const std::string& url)                  // ".../media/t<k>/..."
{
    const size_t at = url.find("media/t");
    return at == std::string::npos ? -1 : atoi(url.c_str() + at + 7);
}
int Streamer::get_url(const char* url, std::vector<uint8_t>& v, uint32_t offset, uint32_t len)
{
    const std::vector<uint8_t>& idx = g_idx[(size_t)title_of(url)];
    v.assign(len, 0);
    for (uint32_t i = 0; i < len && (size_t)offset + i < idx.size(); i++) v[i] = idx[offset + i];
    return (int)len;
}
ssize_t Streamer::read(uint8_t*, uint32_t len, uint32_t*)
{
    if (poster_open() || g_end) { g_run = false; return 0; }    // the end of the stream: the decoder pauses
    return (ssize_t)len;
}
extern "C" void audio_thread(void*) {}
void beep() {}
void clear_events(int e) { if (e & DECODER_RUN) g_run = false; }
void set_events(int e) { if (e & DECODER_RUN) g_run = true; }
void wait_events(int) {}
int get_events() { return g_run ? DECODER_RUN : DECODER_PAUSED; }
void up_key() {}
void down_key() {}
int64_t nv_read(const char* key) { auto it = g_nv.find(key); return it == g_nv.end() ? 0 : it->second; }
void nv_write(const char* key, int64_t pts) { g_nv[key] = pts; g_writes++; }
int printf_nano(const char*, ...) { return 0; }
void push_video(Frame*, int, int64_t, int) {}
int stack() { return 0; }
void start_thread(TaskFunction_t, void*, int) {}
void video_init(int) {}
void video_pause(int) {}
void video_reset() {}
void wifi_disconnect() {}
void wifi_join(const char*, const char*) {}
std::map<std::string, int>& wifi_list() { static std::map<std::string, int> m; return m; }
std::string wifi_ssid() { return std::string(); }
WiFiState wifi_state() { return CONNECTED; }

// the iterations of a script: NEC code, whether the title's read ends there, its step, and whether it is the step's first / last
struct Iter { int nec; bool end; int step; bool first, last; };
static std::vector<Iter> g_iters;
static size_t g_it = 0;
static const int64_t* g_step_pts = nullptr;
static int64_t* g_out = nullptr;
static int g_titles = 0;

// per step: file (0 rwd, 1 main, 2 fwd, 3 poster, -1 none), offset, flush_picture() mode (-1 none), NVS writes, _nav, _speed, _state
// (1 PLAYING, 2 PAUSED, 5 NAV, -1 other), _video_composite_blend, _last_seconds, _info[_nav].pos, then the saved position of every title
static void record(int step)
{
    ESPFlix* p = g_player;
    int64_t* o = g_out + (size_t)step * (10 + g_titles);
    o[0] = g_url.empty() ? -1 : g_url.find("poster.ts") != std::string::npos ? 3 : g_url.find("video_rwd.ts") != std::string::npos ? 0
         : g_url.find("video_fwd.ts") != std::string::npos ? 2 : 1;
    o[1] = o[0] >= 0 ? g_offset : 0;
    o[2] = g_mode;
    o[3] = g_writes;
    o[4] = p->_nav;
    o[5] = p->_speed;
    o[6] = p->_state == ESPFlix::PLAYING ? 1 : p->_state == ESPFlix::PAUSED ? 2 : p->_state == ESPFlix::NAV ? 5 : -1;
    o[7] = _video_composite_blend;
    o[8] = p->_last_seconds;
    o[9] = p->_nav >= 0 ? p->_info[(size_t)p->_nav].pos : 0;
    for (int i = 0; i < g_titles; i++) o[10 + i] = nv_read(p->_manifest[(size_t)i].c_str());
}

int get_nec()
{
    if (g_captured) g_player->_last_seconds = g_capture;   // undo the idle iteration's update_progress()
    g_captured = false;
    if (g_it > 0 && g_iters[g_it - 1].last) record(g_iters[g_it - 1].step);
    if (g_it == g_iters.size()) throw Done();
    const Iter& it = g_iters[g_it++];
    if (it.first) {
        g_pts = g_step_pts[it.step];
        g_url.clear(); g_offset = 0; g_mode = -1; g_writes = 0;
        _video_composite_blend = kSentinel;
        g_player->_last_seconds = kSentinel;
    }
    g_end = it.end;
    return it.nec;
}

extern "C" {

int efref_keys_sentinel() { return kSentinel; }

// a service of n titles t0 .. t<n-1>, their video.idx images back to back (offsets off[n + 1]), connected: init_service()'s nav(0), no
// position saved; then the script's steps (nec[k], ended[k], pts[k]) through loop(). out: n_steps rows of 10 + n int64 (record()).
void efref_keys_run(int n, const uint8_t* idx, const uint64_t* off, int n_steps, const int* nec, const int* ended, const int64_t* pts, int64_t* out)
{
    if (!g_player) g_player = new ESPFlix(1);
    ESPFlix* p = g_player;
    g_idx.clear();
    p->_manifest.clear();
    p->_info.assign((size_t)n, ESPFlix::info());
    for (int i = 0; i < n; i++) {
        g_idx.emplace_back(idx + off[i], idx + off[i + 1]);
        p->_manifest.push_back("t" + std::to_string(i));
        memcpy(&p->_info[(size_t)i].idx, idx + off[i], 104);
    }
    g_nv.clear();
    g_titles = n;
    p->_nav = -1;
    p->_speed = 0;
    p->_state = ESPFlix::NAV;
    p->_pending = ESPFlix::NONE;
    p->_last_seconds = 0;
    p->_gui._wifi_state = CONNECTED;
    g_run = false; g_end = false; g_captured = false;
    p->nav(0);
    g_iters.clear();
    for (int k = 0; k < n_steps; k++) {
        if (ended[k]) g_iters.push_back({ 0, true, k, true, false });
        g_iters.push_back({ nec[k], false, k, !ended[k], false });
        g_iters.push_back({ 0, false, k, false, true });
    }
    g_it = 0;
    g_step_pts = pts;
    g_out = out;
    try {
        p->loop();
    } catch (const Done&) {
    }
}

}  // extern "C"
