// Weight / format plumbing (SURVEY.md section 8f row N4): everything between a checkpoint directory and the b2a_*_create calls.
// Host-only code.  Replaces (reference paths):
//   MLX.loadArrays(url:) on *.safetensors                       (LlamaTTS.swift:982-994 llamaTTSLoadWeights: every file, later wins)
//   WhisperModel.detectFormat / sanitize / sanitizeHuggingFace / sanitizeMlxWhisper / remapMlxWhisperKey / whisperSinusoids
//                                                                (Sources/MLXAudioSTT/Models/Whisper/WhisperModel.swift:315-480)
//   LlamaTTSModel.sanitize (drop rotary inv_freq, drop the tied lm_head)             (LlamaTTS.swift:583-593)
//   quantize(model:) with BaseConfiguration.perLayerQuantization (LlamaTTS.swift:955-966): MLX affine group quantisation.
//     The arithmetic lives in mlx-swift (not on disk); its published format is restated here: weight = uint32 words holding
//     32/bits values each, value j of a word at bits [j*bits, (j+1)*bits); scales / biases [out, in/group_size];
//     w = scales * q + biases.  bits in {2, 4, 8}.  This library computes in bf16, so quantised matrices are expanded to bf16 once
//     at load ("parity unpinned" for this piece: no MLX build here to cross-check; tests pin it to a numpy restatement).
//   config.json decoding (LlamaTTSConfig.swift:100-166, WhisperConfig.swift:78-131): the keys the create calls need.
// A b2a_weights handle keeps the files mapped; tensors are borrowed views unless a sanitiser had to rewrite them.
#include "common.cuh"

#include <dirent.h>
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <cmath>
#include <cctype>
#include <memory>

namespace b2a {

// ------------------------------------------------------------------------------------------------ minimal JSON
struct Json {
    enum Kind { Null, Bool, Num, Str, Arr, Obj } kind = Null;
    bool b = false;
    double num = 0;
    std::string str;
    std::vector<Json> arr;
    std::vector<std::pair<std::string, Json>> obj;
    const Json* find(const std::string& k) const {
        for (auto& kv : obj) if (kv.first == k) return &kv.second;
        return nullptr;
    }
    double number(const std::string& k, double dflt) const {
        const Json* j = find(k);
        return (j && j->kind == Num) ? j->num : (j && j->kind == Bool ? (j->b ? 1.0 : 0.0) : dflt);
    }
    bool has(const std::string& k) const { const Json* j = find(k); return j && j->kind != Null; }
};

struct JsonParser {
    const char* p; const char* end;
    explicit JsonParser(const char* s, size_t n) : p(s), end(s + n) {}
    [[noreturn]] void fail(const char* what) { throw Error(B2A_ERR_MODEL_NOT_INITIALIZED, std::string("json: ") + what); }
    void ws() { while (p < end && (*p == ' ' || *p == '\n' || *p == '\t' || *p == '\r')) ++p; }
    int depth = 0;
    struct Depth { int& d; explicit Depth(int& x) : d(x) { ++d; } ~Depth() { --d; } };
    Json parse() { ws(); Json j = value(); ws(); return j; }
    Json value() {
        Depth guard(depth);
        if (depth > 64) fail("nesting deeper than 64 levels");      // a hostile header must not overflow the stack
        ws();
        if (p >= end) fail("unexpected end");
        Json j;
        if (*p == '{') {
            j.kind = Json::Obj; ++p; ws();
            if (p < end && *p == '}') { ++p; return j; }
            for (;;) {
                ws();
                if (p >= end || *p != '"') fail("expected key");
                std::string k = string();
                ws();
                if (p >= end || *p != ':') fail("expected ':'");
                ++p;
                j.obj.emplace_back(std::move(k), value());
                ws();
                if (p < end && *p == ',') { ++p; continue; }
                if (p < end && *p == '}') { ++p; break; }
                fail("expected ',' or '}'");
            }
        } else if (*p == '[') {
            j.kind = Json::Arr; ++p; ws();
            if (p < end && *p == ']') { ++p; return j; }
            for (;;) {
                j.arr.push_back(value());
                ws();
                if (p < end && *p == ',') { ++p; continue; }
                if (p < end && *p == ']') { ++p; break; }
                fail("expected ',' or ']'");
            }
        } else if (*p == '"') {
            j.kind = Json::Str; j.str = string();
        } else if (!strncmp(p, "true", std::min<size_t>(4, end - p)) && end - p >= 4) { j.kind = Json::Bool; j.b = true; p += 4; }
        else if (!strncmp(p, "false", std::min<size_t>(5, end - p)) && end - p >= 5) { j.kind = Json::Bool; j.b = false; p += 5; }
        else if (!strncmp(p, "null", std::min<size_t>(4, end - p)) && end - p >= 4) { j.kind = Json::Null; p += 4; }
        else {
            char* e = nullptr;
            j.kind = Json::Num; j.num = strtod(p, &e);
            if (e == p) fail("bad value");
            p = e;
        }
        return j;
    }
    std::string string() {
        ++p;
        std::string s;
        while (p < end && *p != '"') {
            if (*p == '\\' && p + 1 < end) {
                ++p;
                switch (*p) {
                    case 'n': s += '\n'; break; case 't': s += '\t'; break; case 'r': s += '\r'; break;
                    case 'b': s += '\b'; break; case 'f': s += '\f'; break;
                    case 'u': { if (end - p < 5) fail("bad escape"); unsigned c = (unsigned)strtoul(std::string(p + 1, 4).c_str(), nullptr, 16);
                                if (c < 0x80) s += (char)c; else s += '?'; p += 4; break; }
                    default: s += *p;
                }
                ++p;
            } else s += *p++;
        }
        if (p >= end) fail("unterminated string");
        ++p;
        return s;
    }
};

static Json read_json_file(const std::string& path) {
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) throw Error(B2A_ERR_MODEL_NOT_INITIALIZED, "cannot open " + path);
    std::string s;
    char buf[65536];
    size_t n;
    while ((n = fread(buf, 1, sizeof buf, f)) > 0) s.append(buf, n);
    fclose(f);
    return JsonParser(s.data(), s.size()).parse();
}

// ------------------------------------------------------------------------------------------------ safetensors
struct Mapped {
    void* base = nullptr; size_t len = 0;
    ~Mapped() { if (base) munmap(base, len); }
};
struct WItem {
    std::string name;
    int dtype = B2A_DTYPE_F32; int ndim = 0; int64_t shape[4] = {0, 0, 0, 0};
    const void* data = nullptr;
    std::shared_ptr<std::vector<uint8_t>> owned;     // set when the bytes were converted / rewritten
    int64_t numel() const { int64_t n = 1; for (int i = 0; i < ndim; ++i) n *= shape[i]; return n; }
};

static float half_to_float(uint16_t h) {
    const uint32_t s = (uint32_t)(h >> 15) << 31, e = (h >> 10) & 0x1f, m = h & 0x3ff;
    uint32_t u;
    if (e == 0) {
        if (m == 0) u = s;
        else { int sh = 0; uint32_t mm = m; while (!(mm & 0x400)) { mm <<= 1; ++sh; } u = s | ((uint32_t)(113 - sh) << 23) | ((mm & 0x3ff) << 13); }
    } else if (e == 31) u = s | 0x7f800000u | (m << 13);
    else u = s | ((e + 112) << 23) | (m << 13);
    float f; memcpy(&f, &u, 4); return f;
}
static float bf16_to_float(uint16_t h) { uint32_t u = (uint32_t)h << 16; float f; memcpy(&f, &u, 4); return f; }
static uint16_t float_to_bf16(float f) {     // round to nearest even (what __float2bfloat16_rn does)
    uint32_t u; memcpy(&u, &f, 4);
    if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);
    u += 0x7fffu + ((u >> 16) & 1u);
    return (uint16_t)(u >> 16);
}

// The "quantization" object of config.json as mlx-swift-lm's BaseConfiguration.PerLayerQuantization reads it (un-vendored; call
// sites LlamaTTSConfig.swift:137-139, LlamaTTS.swift:955-966): group_size / bits are the default, every other key is a layer path
// whose value is either `false` (that layer is not quantised) or its own {group_size, bits}.
struct QuantSpec {
    int group_size = 0, bits = 0;
    std::map<std::string, std::pair<int, int>> per_layer;
    std::vector<std::string> off;
    bool any() const { return bits > 0 || !per_layer.empty(); }
    // 1 = quantised with (gs, b); 0 = no setting for this layer
    int lookup(const std::string& path, int& gs, int& b) const {
        for (auto& o : off) if (o == path) return 0;
        auto it = per_layer.find(path);
        if (it != per_layer.end()) { gs = it->second.first; b = it->second.second; return 1; }
        if (bits > 0) { gs = group_size; b = bits; return 1; }
        return 0;
    }
};
static QuantSpec parse_quant(const Json& cfg) {
    QuantSpec q;
    const Json* j = cfg.find("quantization");
    if (!j || j->kind != Json::Obj) return q;
    q.group_size = (int)j->number("group_size", 64);
    q.bits = (int)j->number("bits", 4);
    for (auto& kv : j->obj) {
        if (kv.first == "group_size" || kv.first == "bits" || kv.first == "mode") continue;
        if (kv.second.kind == Json::Bool && !kv.second.b) q.off.push_back(kv.first);
        else if (kv.second.kind == Json::Obj)
            q.per_layer[kv.first] = {(int)kv.second.number("group_size", q.group_size), (int)kv.second.number("bits", q.bits)};
    }
    return q;
}

}  // namespace b2a

using namespace b2a;

struct b2a_weights {
    std::vector<std::shared_ptr<Mapped>> maps;
    std::vector<WItem> items;

    int find(const std::string& n) const {
        for (size_t i = 0; i < items.size(); ++i) if (items[i].name == n) return (int)i;
        return -1;
    }
    void put(WItem&& it) {
        const int i = find(it.name);
        if (i >= 0) items[i] = std::move(it); else items.push_back(std::move(it));     // later files win (weights.merge { _, new in new })
    }
    void erase(const std::string& n) { const int i = find(n); if (i >= 0) items.erase(items.begin() + i); }

    void load_file(const std::string& path) {
        const int fd = open(path.c_str(), O_RDONLY);
        B2A_CHECK(fd >= 0, B2A_ERR_MODEL_NOT_INITIALIZED, "cannot open " + path);
        struct stat st{};
        fstat(fd, &st);
        auto mp = std::make_shared<Mapped>();
        mp->len = (size_t)st.st_size;
        B2A_CHECK(mp->len >= 8, B2A_ERR_MODEL_NOT_INITIALIZED, "not a safetensors file: " + path);
        mp->base = mmap(nullptr, mp->len, PROT_READ, MAP_PRIVATE, fd, 0);
        close(fd);
        B2A_CHECK(mp->base != MAP_FAILED, B2A_ERR_MODEL_NOT_INITIALIZED, "mmap failed: " + path);
        const uint8_t* b = (const uint8_t*)mp->base;
        uint64_t hl; memcpy(&hl, b, 8);
        B2A_CHECK(hl <= mp->len - 8, B2A_ERR_MODEL_NOT_INITIALIZED, "corrupt safetensors header: " + path);
        Json hdr = JsonParser((const char*)b + 8, (size_t)hl).parse();
        B2A_CHECK(hdr.kind == Json::Obj, B2A_ERR_MODEL_NOT_INITIALIZED, "corrupt safetensors header: " + path);
        const uint8_t* data = b + 8 + hl;
        const size_t data_len = mp->len - 8 - (size_t)hl;
        maps.push_back(mp);
        for (auto& kv : hdr.obj) {
            if (kv.first == "__metadata__") continue;
            const Json& t = kv.second;
            const Json* dt = t.find("dtype"); const Json* sh = t.find("shape"); const Json* off = t.find("data_offsets");
            B2A_CHECK(dt && sh && off && off->arr.size() == 2, B2A_ERR_MODEL_NOT_INITIALIZED, "corrupt tensor entry: " + kv.first);
            WItem it;
            it.name = kv.first;
            it.ndim = (int)sh->arr.size();
            B2A_CHECK(it.ndim <= 4, B2A_ERR_MODEL_NOT_INITIALIZED, "more than 4 dimensions: " + kv.first);
            int64_t total = 1;
            for (int i = 0; i < it.ndim; ++i) {
                const double d = sh->arr[i].num;
                B2A_CHECK(sh->arr[i].kind == Json::Num && d >= 0 && d <= 9.0e15 && d == (double)(int64_t)d, B2A_ERR_MODEL_NOT_INITIALIZED,
                          "safetensors: shape entries must be non-negative integers: " + it.name);
                it.shape[i] = (int64_t)d;
                B2A_CHECK(it.shape[i] == 0 || total <= ((int64_t)1 << 46) / it.shape[i], B2A_ERR_MODEL_NOT_INITIALIZED,
                          "safetensors: tensor too large: " + it.name);            // numel() cannot overflow below
                total *= it.shape[i];
            }
            const size_t o0 = (size_t)off->arr[0].num, o1 = (size_t)off->arr[1].num;
            B2A_CHECK(o0 <= o1 && o1 <= data_len, B2A_ERR_MODEL_NOT_INITIALIZED, "tensor out of bounds: " + kv.first);
            const uint8_t* src = data + o0;
            const int64_t n = it.numel();
            const std::string& d = dt->str;
            auto need = [&](size_t esz) { B2A_CHECK((size_t)n * esz == o1 - o0, B2A_ERR_MODEL_NOT_INITIALIZED, "size mismatch: " + kv.first); };
            if (d == "F32") { need(4); it.dtype = B2A_DTYPE_F32; it.data = src; }
            else if (d == "BF16") { need(2); it.dtype = B2A_DTYPE_BF16; it.data = src; }
            else if (d == "I32" || d == "U32") { need(4); it.dtype = B2A_DTYPE_I32; it.data = src; }
            else if (d == "F16") {
                need(2);
                it.owned = std::make_shared<std::vector<uint8_t>>((size_t)n * 4);
                float* o = (float*)it.owned->data();
                const uint16_t* s16 = (const uint16_t*)src;
                for (int64_t i = 0; i < n; ++i) o[i] = half_to_float(s16[i]);
                it.dtype = B2A_DTYPE_F32; it.data = o;
            } else if (d == "I64") {
                need(8);
                it.owned = std::make_shared<std::vector<uint8_t>>((size_t)n * 4);
                int32_t* o = (int32_t*)it.owned->data();
                const int64_t* s64 = (const int64_t*)src;
                for (int64_t i = 0; i < n; ++i) o[i] = (int32_t)s64[i];
                it.dtype = B2A_DTYPE_I32; it.data = o;
            } else {
                throw Error(B2A_ERR_MODEL_NOT_INITIALIZED, "unsupported safetensors dtype " + d + " for " + kv.first);
            }
            put(std::move(it));
        }
    }

    void load(const std::string& path) {
        struct stat st{};
        B2A_CHECK(stat(path.c_str(), &st) == 0, B2A_ERR_MODEL_NOT_INITIALIZED, "no such file or directory: " + path);
        if (!S_ISDIR(st.st_mode)) { load_file(path); return; }
        std::vector<std::string> files;
        DIR* d = opendir(path.c_str());
        B2A_CHECK(d, B2A_ERR_MODEL_NOT_INITIALIZED, "cannot list " + path);
        while (dirent* e = readdir(d)) {
            const std::string n = e->d_name;
            if (n.size() > 12 && n.substr(n.size() - 12) == ".safetensors") files.push_back(path + "/" + n);
        }
        closedir(d);
        B2A_CHECK(!files.empty(), B2A_ERR_MODEL_NOT_INITIALIZED, "no .safetensors file in " + path);
        std::sort(files.begin(), files.end());
        for (auto& f : files) load_file(f);
    }

    std::vector<float> as_f32(const WItem& t) const {
        const int64_t n = t.numel();
        std::vector<float> v((size_t)n);
        if (t.dtype == B2A_DTYPE_F32) memcpy(v.data(), t.data, (size_t)n * 4);
        else if (t.dtype == B2A_DTYPE_BF16) { const uint16_t* s = (const uint16_t*)t.data; for (int64_t i = 0; i < n; ++i) v[i] = bf16_to_float(s[i]); }
        else throw Error(B2A_ERR_MODEL_NOT_INITIALIZED, "expected a floating-point tensor: " + t.name);
        return v;
    }

    // ---- Whisper (WhisperModel.swift:315-480).  Output: HF (`transformers`) names with the `model.` prefix and conv weights in the
    // PyTorch [out, in, k] layout -- what b2a_stt_create takes (the reference moves them to MLX's [out, k, in] instead).
    static bool strip(const std::string& s, const std::string& pre, std::string& rest) {
        if (s.compare(0, pre.size(), pre) != 0) return false;
        rest = s.substr(pre.size());
        return true;
    }
    static bool remap_attn(const std::string& suffix, const std::string& container, std::string& out) {
        const size_t dot = suffix.find('.');
        if (dot == std::string::npos) return false;
        const std::string which = suffix.substr(0, dot), rest = suffix.substr(dot + 1);
        const char* m = which == "query" ? "q_proj" : which == "key" ? "k_proj" : which == "value" ? "v_proj" : which == "out" ? "out_proj" : nullptr;
        if (!m) return false;
        out = container + "." + m + "." + rest;
        return true;
    }
    static bool remap_block(const std::string& suffix, bool dec, std::string& out) {
        std::string r;
        if (strip(suffix, "attn_ln.", r)) { out = "self_attn_layer_norm." + r; return true; }
        if (dec && strip(suffix, "cross_attn_ln.", r)) { out = "encoder_attn_layer_norm." + r; return true; }
        if (strip(suffix, "mlp_ln.", r)) { out = "final_layer_norm." + r; return true; }
        if (strip(suffix, "mlp1.", r)) { out = "fc1." + r; return true; }
        if (strip(suffix, "mlp2.", r)) { out = "fc2." + r; return true; }
        if (strip(suffix, "attn.", r)) return remap_attn(r, "self_attn", out);
        if (dec && strip(suffix, "cross_attn.", r)) return remap_attn(r, "encoder_attn", out);
        return false;
    }
    static bool remap_mlx_whisper(const std::string& k, std::string& out) {
        std::string r;
        if (k == "encoder.positional_embedding") { out = "model.encoder.embed_positions.weight"; return true; }
        if (k == "decoder.positional_embedding") { out = "model.decoder.embed_positions.weight"; return true; }
        if (strip(k, "decoder.token_embedding.", r)) { out = "model.decoder.embed_tokens." + r; return true; }
        if (k == "encoder.conv1.weight" || k == "encoder.conv1.bias" || k == "encoder.conv2.weight" || k == "encoder.conv2.bias") { out = "model." + k; return true; }
        if (strip(k, "encoder.ln_post.", r)) { out = "model.encoder.layer_norm." + r; return true; }
        if (strip(k, "decoder.ln.", r)) { out = "model.decoder.layer_norm." + r; return true; }
        for (const char* stem : {"encoder", "decoder"}) {
            if (!strip(k, std::string(stem) + ".blocks.", r)) continue;
            const size_t dot = r.find('.');
            if (dot == std::string::npos) return false;
            std::string mapped;
            if (!remap_block(r.substr(dot + 1), std::string(stem) == "decoder", mapped)) return false;
            out = std::string("model.") + stem + ".layers." + r.substr(0, dot) + "." + mapped;
            return true;
        }
        return false;
    }
    void transpose_12(WItem& t) {    // [a, b, c] -> [a, c, b]
        std::vector<float> v = as_f32(t);
        const int64_t A = t.shape[0], Bd = t.shape[1], Cd = t.shape[2];
        auto o = std::make_shared<std::vector<uint8_t>>((size_t)(A * Bd * Cd) * 4);
        float* of = (float*)o->data();
        for (int64_t a = 0; a < A; ++a)
            for (int64_t b = 0; b < Bd; ++b)
                for (int64_t c = 0; c < Cd; ++c) of[(a * Cd + c) * Bd + b] = v[(a * Bd + b) * Cd + c];
        t.owned = o; t.data = of; t.dtype = B2A_DTYPE_F32; t.shape[1] = Cd; t.shape[2] = Bd;
    }
    int sanitize_whisper() {     // returns 0 = huggingFace, 1 = mlxWhisper (detectFormat :321-326)
        bool mlx = false;
        for (auto& it : items) if (it.name.find(".blocks.") != std::string::npos) { mlx = true; break; }
        std::vector<WItem> out;
        if (!mlx) {
            for (auto& it : items) {
                if (it.name == "proj_out.weight" || it.name == "model.proj_out.weight") continue;       // tied to embed_tokens (:338-342)
                WItem t = it;
                if (t.name.compare(0, 6, "model.") != 0 && (t.name.compare(0, 8, "encoder.") == 0 || t.name.compare(0, 8, "decoder.") == 0))
                    t.name = "model." + t.name;
                out.push_back(std::move(t));
            }
        } else {
            for (auto& it : items) {
                if (it.name == "alignment_heads") continue;
                std::string mapped;
                if (!remap_mlx_whisper(it.name, mapped)) continue;
                WItem t = it;
                t.name = mapped;
                if ((mapped == "model.encoder.conv1.weight" || mapped == "model.encoder.conv2.weight") && t.ndim == 3)
                    transpose_12(t);                                      // MLX [out, k, in] -> PyTorch [out, in, k]
                out.push_back(std::move(t));
            }
        }
        items = std::move(out);
        // mlx-whisper omits the fixed sinusoidal encoder positions (:370-376, whisperSinusoids :381-395)
        if (find("model.encoder.embed_positions.weight") < 0) {
            const int c2 = find("model.encoder.conv2.weight");
            if (c2 >= 0) {
                const int64_t ch = items[c2].shape[0], len = 1500, half = ch / 2;
                B2A_CHECK(ch % 2 == 0, B2A_ERR_MODEL_NOT_INITIALIZED, "Whisper sinusoid channels must be even");
                auto o = std::make_shared<std::vector<uint8_t>>((size_t)(len * ch) * 4);
                float* v = (float*)o->data();
                const double inc = std::log(10000.0) / (double)std::max<int64_t>(half - 1, 1);
                for (int64_t pos = 0; pos < len; ++pos)
                    for (int64_t i = 0; i < half; ++i) {
                        const double st = (double)pos * std::exp(-inc * (double)i);
                        v[pos * ch + i] = (float)std::sin(st);
                        v[pos * ch + half + i] = (float)std::cos(st);
                    }
                WItem t; t.name = "model.encoder.embed_positions.weight"; t.dtype = B2A_DTYPE_F32; t.ndim = 2; t.shape[0] = len; t.shape[1] = ch;
                t.owned = o; t.data = v;
                items.push_back(std::move(t));
            }
        }
        return mlx ? 1 : 0;
    }

    // ---- Llama / Orpheus (LlamaTTS.swift:583-593 sanitize, :955-966 quantize)
    void sanitize_llama(bool tie, int group_size, int bits) {
        QuantSpec q;
        q.group_size = group_size; q.bits = bits;
        sanitize_llama(tie, q);
    }
    void sanitize_llama(bool tie, const QuantSpec& spec) {
        std::vector<WItem> out;
        for (auto& it : items) {
            if (it.name.find("self_attn.rotary_emb.inv_freq") != std::string::npos) continue;
            if (tie && it.name == "lm_head.weight") continue;
            out.push_back(it);
        }
        items = std::move(out);
        dequantize_layers(spec);
    }
    // MLX affine de-quantisation of every layer that carries "<path>.scales" (the reference tests weights["\(path).scales"],
    // LlamaTTS.swift:958-962; Whisper quantises every Linear and decoder.embed_tokens, WhisperModel.swift:499-511): w = scales * q + biases,
    // value j of a uint32 word at bits [j * bits, (j + 1) * bits), result stored as bf16.
    void dequantize_layers(const QuantSpec& spec) {
        if (!spec.any()) return;
        std::vector<std::string> paths;
        for (auto& it : items) {
            const size_t n = it.name.size();
            if (n > 7 && it.name.substr(n - 7) == ".scales") paths.push_back(it.name.substr(0, n - 7));
        }
        for (auto& p : paths) {
            int group_size = 0, bits = 0;
            B2A_CHECK(spec.lookup(p, group_size, bits) == 1, B2A_ERR_MODEL_NOT_INITIALIZED, "quantised tensors for a layer the config does not quantise: " + p);
            B2A_CHECK(bits == 2 || bits == 4 || bits == 8, B2A_ERR_INVALID_INPUT, "MLX affine quantisation: bits must be 2, 4 or 8");
            B2A_CHECK(group_size > 0 && group_size % (32 / bits) == 0, B2A_ERR_INVALID_INPUT, "MLX affine quantisation: bad group_size");
            const int iw = find(p + ".weight"), is = find(p + ".scales"), ib = find(p + ".biases");
            B2A_CHECK(iw >= 0 && is >= 0 && ib >= 0, B2A_ERR_MODEL_NOT_INITIALIZED, "incomplete quantised layer: " + p);
            const WItem& w = items[iw];
            B2A_CHECK(w.dtype == B2A_DTYPE_I32 && w.ndim == 2, B2A_ERR_MODEL_NOT_INITIALIZED, "quantised weight must be uint32 [out, in*bits/32]: " + p);
            const int per = 32 / bits;
            const int64_t rows = w.shape[0], words = w.shape[1], cols = words * per, groups = cols / group_size;
            B2A_CHECK(cols % group_size == 0, B2A_ERR_MODEL_NOT_INITIALIZED, "quantised weight: columns are not a multiple of group_size: " + p);
            const std::vector<float> sc = as_f32(items[is]), bi = as_f32(items[ib]);
            B2A_CHECK((int64_t)sc.size() == rows * groups && bi.size() == sc.size(), B2A_ERR_MODEL_NOT_INITIALIZED, "bad scales / biases shape: " + p);
            auto o = std::make_shared<std::vector<uint8_t>>((size_t)(rows * cols) * 2);
            uint16_t* dst = (uint16_t*)o->data();
            const uint32_t* q = (const uint32_t*)w.data;
            const uint32_t mask = (1u << bits) - 1u;
            for (int64_t r = 0; r < rows; ++r)
                for (int64_t c = 0; c < cols; ++c) {
                    const uint32_t word = q[r * words + c / per];
                    const float v = (float)((word >> ((c % per) * bits)) & mask);
                    const int64_t g = r * groups + c / group_size;
                    dst[r * cols + c] = float_to_bf16(fmaf(sc[g], v, bi[g]));
                }
            WItem t; t.name = p + ".weight"; t.dtype = B2A_DTYPE_BF16; t.ndim = 2; t.shape[0] = rows; t.shape[1] = cols; t.owned = o; t.data = dst;
            items[iw] = std::move(t);
            erase(p + ".scales"); erase(p + ".biases");
        }
    }

    // ---- Soprano: SopranoModel.sanitize (Soprano.swift:314-361), then the MLX de-quantisation of every layer with ".scales"
    // (:950-963).  decoder.* keeps its keys (b2a_soprano_create hands them to the Vocos decoder, which reads them as fp32).
    void sanitize_soprano(bool tie, const QuantSpec& spec) {
        std::vector<WItem> out;
        for (auto& it : items) {
            WItem t = it;
            std::string k = it.name;
            if (k.rfind("model.", 0) == 0) k = k.substr(6);                    // "model.language_model.*" -> "language_model.*"
            if (k.rfind("decoder.", 0) == 0) {
            } else if (k.rfind("language_model.lm_head", 0) == 0) {
                k = k.substr(15);                                               // lm_head sits on SopranoModel itself
            } else if (k.rfind("language_model.", 0) == 0) {
                k = "model." + k.substr(15);
            } else if (k.rfind("lm_head", 0) != 0) {
                k = "model." + k;                                               // bare inner keys: embed_tokens.*, layers.*, norm.*
            }
            if (tie && k == "lm_head.weight") continue;
            t.name = k;
            out.push_back(std::move(t));
        }
        items.clear();
        for (auto& t : out) put(std::move(t));
        dequantize_layers(spec);
    }

    // ---- Qwen3-TTS talker: Qwen3TTSTalkerForConditionalGeneration.sanitize (Qwen3TTSTalker.swift:356-365) keeps "talker.*" and drops
    // the prefix; a quantised checkpoint (config "quantization", Qwen3TTS.swift:1156-1171: every layer that carries ".scales") is
    // expanded to bf16 -- the engine streams bf16 matrices.
    void sanitize_qwen3_talker(const QuantSpec& spec) {
        std::vector<WItem> out;
        for (auto& it : items) {
            if (it.name.rfind("talker.", 0) != 0) continue;
            WItem t = it;
            t.name = it.name.substr(7);
            out.push_back(std::move(t));
        }
        items = std::move(out);
        dequantize_layers(spec);
    }

    // ---- Qwen3-TTS speech tokenizer, decoder half of Qwen3TTSSpeechTokenizer.sanitize (Qwen3TTSSpeechTokenizer.swift:1094-1440).
    // Output: the keys b2a_speech_tokenizer_create takes (below the "decoder." module) in MLX layouts.  encoder.* (voice-cloning
    // encoder) and speaker-encoder keys are dropped.
    static bool check_array_shape(const WItem& t) {      // checkArrayShapeQwen3 (:1445-1455)
        if (t.ndim != 3) return false;
        const int64_t d2 = t.shape[1], d3 = t.shape[2];
        if (d2 == 1) return d3 > 64;
        if (d3 == 1) return d2 <= 64;
        return d2 < d3;
    }
    void permute3(WItem& t, int p0, int p1, int p2) {    // out[i, j, k] = in[index with out axis a taken from in axis p_a]
        std::vector<float> v = as_f32(t);
        const int64_t in_shape[3] = {t.shape[0], t.shape[1], t.shape[2]};
        const int p[3] = {p0, p1, p2};
        const int64_t o0 = in_shape[p0], o1 = in_shape[p1], o2 = in_shape[p2];
        const int64_t in_stride[3] = {in_shape[1] * in_shape[2], in_shape[2], 1};
        auto o = std::make_shared<std::vector<uint8_t>>((size_t)(o0 * o1 * o2) * 4);
        float* of = (float*)o->data();
        for (int64_t a = 0; a < o0; ++a)
            for (int64_t b = 0; b < o1; ++b)
                for (int64_t c = 0; c < o2; ++c)
                    of[(a * o1 + b) * o2 + c] = v[a * in_stride[p[0]] + b * in_stride[p[1]] + c * in_stride[p[2]]];
        t.owned = o; t.data = of; t.dtype = B2A_DTYPE_F32; t.shape[0] = o0; t.shape[1] = o1; t.shape[2] = o2;
    }
    static bool has_component_with_suffix(const std::string& key, const std::string& comp) {     // stripSpeakerEncoderPrefix != nil (Qwen3TTSSpeakerEncoder.swift:345-354)
        size_t pos = 0;
        while (pos <= key.size()) {
            const size_t dot = key.find('.', pos);
            const std::string part = key.substr(pos, dot == std::string::npos ? std::string::npos : dot - pos);
            if (part == comp) return dot != std::string::npos && dot + 1 < key.size();
            if (dot == std::string::npos) break;
            pos = dot + 1;
        }
        return false;
    }
    void sanitize_speech_tokenizer() {
        std::vector<WItem> out;
        std::vector<std::pair<std::string, WItem>> usage, sums;
        for (auto& it : items) {
            std::string k = it.name;
            for (bool stripped = true; stripped;) {                   // stripKnownPrefixes (:1118-1133)
                stripped = false;
                for (const char* pre : {"speech_tokenizer.", "encoder_model.", "decoder_model."}) {
                    std::string rest;
                    if (strip(k, pre, rest)) { k = rest; stripped = true; break; }
                }
            }
            if (k.empty() || k == "encoder_model" || k == "decoder_model" || k == "speech_tokenizer") continue;
            if (has_component_with_suffix(k, "speaker_encoder")) continue;
            const bool cu = k.find("_codebook.cluster_usage") != std::string::npos, es = k.find("_codebook.embedding_sum") != std::string::npos;
            if (cu || es) {                                           // :1226-1235
                WItem t = it;
                const std::string base = k.substr(0, k.rfind("._codebook."));
                (cu ? usage : sums).emplace_back(base, std::move(t));
                continue;
            }
            if (k.find("_codebook.initialized") != std::string::npos || k.find(".codebook.initialized") != std::string::npos) continue;
            if (k.compare(0, 8, "encoder.") == 0) continue;
            WItem t = it;
            const bool tconv = (k.find("upsample") != std::string::npos && k.find(".0.conv.weight") != std::string::npos) ||
                               (k.find("decoder.decoder") != std::string::npos && k.find("block.1.conv.weight") != std::string::npos);
            if (t.ndim == 3) {
                if (tconv) { if (!check_array_shape(t)) permute3(t, 1, 2, 0); }                      // torch [in, out, k] -> [out, k, in]
                else if (k.find("conv.weight") != std::string::npos || k.find("_proj.weight") != std::string::npos) {
                    if (!check_array_shape(t)) permute3(t, 0, 2, 1);                                  // torch [out, in, k] -> [out, k, in]
                }
            }
            // upsample.X.Y.rest -> upsample.X.layers.Y.rest (:1406-1413)
            const size_t u = k.find("upsample.");
            if (u != std::string::npos) {
                size_t a = u + 9, b = a;
                while (b < k.size() && isdigit((unsigned char)k[b])) ++b;
                if (b > a && b < k.size() && k[b] == '.') {
                    size_t c = b + 1, d = c;
                    while (d < k.size() && isdigit((unsigned char)k[d])) ++d;
                    if (d > c) k = k.substr(0, b + 1) + "layers." + k.substr(c);
                }
            }
            t.name = k;
            out.push_back(std::move(t));
        }
        for (auto& u : usage)
            for (auto& e : sums)
                if (e.first == u.first) {                             // both statistics present (:1431-1438)
                    WItem a = u.second, b = e.second;
                    a.name = u.first + ".codebook.cluster_usage";
                    b.name = u.first + ".codebook.embedding_sum";
                    out.push_back(std::move(a));
                    out.push_back(std::move(b));
                }
        for (auto& t : out) {                                         // the decoder module's own keys
            std::string rest;
            if (strip(t.name, "decoder.", rest) && !(rest.size() && isdigit((unsigned char)rest[0]))) t.name = rest;
        }
        items = std::move(out);
    }

    // ---- Qwen3-TTS speech tokenizer, encoder half of Qwen3TTSSpeechTokenizer.sanitize (Qwen3TTSSpeechTokenizer.swift:1093-1440).
    // Output: the keys b2a_speech_tokenizer_encoder_create takes -- the reference's "encoder_model." paths without that prefix -- in
    // MLX layouts.  Every non-encoder key is dropped; the codebooks' "initialized" flags are not emitted (nothing reads them).
    static WItem f32_item(const std::string& name, std::vector<float>&& v, int64_t rows, int64_t cols) {
        WItem t;
        auto o = std::make_shared<std::vector<uint8_t>>(v.size() * 4);
        memcpy(o->data(), v.data(), v.size() * 4);
        t.name = name; t.owned = o; t.data = o->data(); t.dtype = B2A_DTYPE_F32; t.ndim = 2; t.shape[0] = rows; t.shape[1] = cols;
        return t;
    }
    void sanitize_speech_tokenizer_encoder() {
        static const std::map<int, std::string> conv_map = {{0, "encoder.init_conv1d"}, {3, "encoder.layers.0.downsample"},
                                                            {6, "encoder.layers.1.downsample"}, {9, "encoder.layers.2.downsample"},
                                                            {12, "encoder.layers.3.downsample"}, {14, "encoder.final_conv1d"}};
        static const std::map<int, int> res_layer = {{1, 0}, {4, 1}, {7, 2}, {10, 3}}, res_block = {{1, 0}, {3, 1}};
        auto split = [](const std::string& k) {
            std::vector<std::string> p;
            size_t a = 0;
            for (size_t b; (b = k.find('.', a)) != std::string::npos; a = b + 1) p.push_back(k.substr(a, b - a));
            p.push_back(k.substr(a));
            return p;
        };
        auto join_from = [](const std::vector<std::string>& p, size_t i) {
            std::string s;
            for (; i < p.size(); ++i) s += (s.empty() ? "" : ".") + p[i];
            return s;
        };
        auto to_int = [](const std::string& s, int& v) {
            if (s.empty() || s.size() > 9) return false;
            for (char c : s) if (!isdigit((unsigned char)c)) return false;
            v = atoi(s.c_str());
            return true;
        };
        auto ends_with = [](const std::string& s, const std::string& e) { return s.size() >= e.size() && s.compare(s.size() - e.size(), e.size(), e) == 0; };
        auto has = [](const std::string& s, const char* x) { return s.find(x) != std::string::npos; };
        auto quant_prefix = [&](const std::string& r, bool contains) {      // mapEncoderQuantizerPrefix / encoderCodebookPrefix
            auto test = [&](const char* x) { return contains ? has(r, x) : r.rfind(x, 0) == 0; };
            if (test("semantic_residual_vector_quantizer") || test("rvq_first.")) return std::string("quantizer.rvq_first");
            return std::string("quantizer.rvq_rest");
        };
        std::vector<WItem> out;
        std::map<int, std::map<char, WItem>> qkv;
        std::map<std::string, std::map<std::string, WItem>> books;
        for (auto& it : items) {
            std::string k = it.name;
            for (bool stripped = true; stripped;) {
                stripped = false;
                for (const char* pre : {"speech_tokenizer.", "encoder_model.", "decoder_model."}) {
                    std::string rest;
                    if (strip(k, pre, rest)) { k = rest; stripped = true; break; }
                }
            }
            if (k.empty() || k == "encoder_model" || k == "decoder_model" || k == "speech_tokenizer") continue;
            if (has_component_with_suffix(k, "speaker_encoder")) continue;
            if (has(k, "_codebook.cluster_usage") || has(k, "_codebook.embedding_sum")) continue;        // the decoder's codebooks
            if (has(k, "_codebook.initialized") || has(k, ".codebook.initialized")) continue;
            if (k.rfind("encoder.", 0) != 0) continue;
            WItem t = it;
            const std::vector<std::string> parts = split(k);
            if (k.rfind("encoder.encoder.layers.", 0) == 0) {                                           // :1241-1269
                int n = 0;
                if (parts.size() < 4 || !to_int(parts[3], n)) continue;
                std::string key;
                if (has(k, ".block.")) {
                    int blk = 0;
                    if (!res_layer.count(n) || parts.size() <= 5 || !to_int(parts[5], blk) || !res_block.count(blk)) continue;
                    key = "encoder.layers." + std::to_string(res_layer.at(n)) + ".residuals.0.block." + std::to_string(res_block.at(blk)) + ".conv." + join_from(parts, 6);
                } else if (conv_map.count(n)) {
                    key = conv_map.at(n) + ".conv." + join_from(parts, 4);
                } else {
                    continue;
                }
                if (ends_with(key, "weight") && t.ndim == 3) permute3(t, 0, 2, 1);
                t.name = key;
                out.push_back(std::move(t));
                continue;
            }
            if (k.rfind("encoder.encoder_transformer.layers.", 0) == 0 || k.rfind("encoder.encoder_transformer.transformer.layers.", 0) == 0) {   // :1271-1322
                const bool nested = parts.size() >= 5 && parts[2] == "transformer" && parts[3] == "layers";
                const size_t off = nested ? 4 : 3;
                int l = 0;
                if (parts.size() <= off || !to_int(parts[off], l)) continue;
                const std::string sfx = join_from(parts, off + 1), p = "encoder_transformer.transformer.layers." + std::to_string(l) + ".";
                std::string key;
                if (has(sfx, "self_attn.q_proj.weight")) { qkv[l]['q'] = t; continue; }
                else if (has(sfx, "self_attn.k_proj.weight")) { qkv[l]['k'] = t; continue; }
                else if (has(sfx, "self_attn.v_proj.weight")) { qkv[l]['v'] = t; continue; }
                else if (has(sfx, "self_attn.qkv.weight") && t.ndim == 2) {
                    const int64_t rows = t.shape[0], cols = t.shape[1], third = rows / 3;
                    if (rows % 3 != 0 || third <= 0) continue;
                    const std::vector<float> v = as_f32(t);
                    const char names[3] = {'q', 'k', 'v'};
                    for (int i = 0; i < 3; ++i)
                        qkv[l][names[i]] = f32_item("", std::vector<float>(v.begin() + i * third * cols, v.begin() + (i + 1) * third * cols), third, cols);
                    continue;
                }
                else if (has(sfx, "self_attn.out_proj.weight") || has(sfx, "self_attn.o_proj.weight")) key = p + "self_attn.out_proj.weight";
                else if (has(sfx, "mlp.fc1.weight")) key = p + "gating.linear1.weight";
                else if (has(sfx, "mlp.fc2.weight")) key = p + "gating.linear2.weight";
                else if (has(sfx, "input_layernorm.weight")) key = p + "norm1.weight";
                else if (has(sfx, "input_layernorm.bias")) key = p + "norm1.bias";
                else if (has(sfx, "post_attention_layernorm.weight")) key = p + "norm2.weight";
                else if (has(sfx, "post_attention_layernorm.bias")) key = p + "norm2.bias";
                else if (has(sfx, "self_attn_layer_scale.scale")) key = p + "layer_scale_1.scale";
                else if (has(sfx, "mlp_layer_scale.scale")) key = p + "layer_scale_2.scale";
                else continue;
                t.name = key;
                out.push_back(std::move(t));
                continue;
            }
            if (k.rfind("encoder.downsample.", 0) == 0) {                                                 // :1324-1332
                const std::string sfx = k.substr(19);
                if (ends_with(sfx, "weight") && t.ndim == 3) permute3(t, 0, 2, 1);
                t.name = "downsample.conv.conv." + sfx;
                out.push_back(std::move(t));
                continue;
            }
            if (k.rfind("encoder.quantizer.", 0) == 0) {                                                  // :1334-1376
                const std::string rest = k.substr(18);
                if (has(rest, ".codebook.embed.weight") || ends_with(rest, "codebook.embed")) continue;
                if (has(rest, "codebook.cluster_usage") || has(rest, "codebook.embed_sum") || has(rest, "codebook.embedding_sum")) {
                    const std::string base = rest.substr(0, rest.rfind(".codebook.") == std::string::npos ? rest.size() : rest.rfind(".codebook."));
                    books[base][has(rest, "cluster_usage") ? "cluster_usage" : "embedding_sum"] = t;
                    continue;
                }
                if (has(rest, "codebook.initialized")) continue;
                if (has(rest, "input_proj.weight") || has(rest, "output_proj.weight")) {
                    if (ends_with(rest, "weight") && t.ndim == 3) permute3(t, 0, 2, 1);
                    WItem c = t;
                    c.name = quant_prefix(rest, false) + (has(rest, "input_proj") ? ".input_proj.weight" : ".output_proj.weight");
                    out.push_back(std::move(c));
                }
                if (!has(rest, "codebook.") && (rest.rfind("layers.", 0) == 0 || has(rest, ".layers."))) {   // mapEncoderQuantizerLayers
                    std::string key;
                    for (const char* pre : {"rvq_first.", "rvq_rest.", "semantic_residual_vector_quantizer.", "acoustic_residual_vector_quantizer."})
                        if (key.empty() && rest.rfind(pre, 0) == 0)
                            key = std::string(pre[0] == 's' || pre[4] == 'f' ? "quantizer.rvq_first.vq." : "quantizer.rvq_rest.vq.") + rest.substr(strlen(pre));
                    if (key.empty() && rest.rfind("layers.", 0) == 0) key = "quantizer.rvq_rest.vq." + rest;
                    if (!key.empty()) { t.name = key; out.push_back(std::move(t)); }
                }
                continue;
            }
        }
        for (auto& e : qkv) {                                                                               // :1397-1401
            auto& m = e.second;
            if (!m.count('q') || !m.count('k') || !m.count('v')) continue;
            std::vector<float> w = as_f32(m['q']), kk = as_f32(m['k']), vv = as_f32(m['v']);
            const int64_t cols = m['q'].ndim == 2 ? m['q'].shape[1] : 0;
            B2A_CHECK(cols > 0 && m['k'].ndim == 2 && m['v'].ndim == 2 && m['k'].shape[1] == cols && m['v'].shape[1] == cols, B2A_ERR_MODEL_NOT_INITIALIZED,
                      "bad shape for tensor: speech tokenizer encoder q / k / v projection");
            const int64_t rows = m['q'].shape[0] + m['k'].shape[0] + m['v'].shape[0];
            w.insert(w.end(), kk.begin(), kk.end());
            w.insert(w.end(), vv.begin(), vv.end());
            out.push_back(f32_item("encoder_transformer.transformer.layers." + std::to_string(e.first) + ".self_attn.in_proj.weight", std::move(w), rows, cols));
        }
        for (auto& e : books) {                                                                             // :1403-1419
            if (!e.second.count("cluster_usage") || !e.second.count("embedding_sum")) continue;
            const std::vector<std::string> parts = split(e.first);
            int idx = -1;
            for (size_t i = 0; i + 1 < parts.size(); ++i)
                if (parts[i] == "layers") { if (!to_int(parts[i + 1], idx)) idx = -1; break; }
            if (idx < 0) continue;
            const std::string p = quant_prefix(e.first, true) + ".vq.layers." + std::to_string(idx) + ".codebook.";
            WItem a = e.second["cluster_usage"], b = e.second["embedding_sum"];
            a.name = p + "cluster_usage"; b.name = p + "embedding_sum";
            out.push_back(std::move(a));
            out.push_back(std::move(b));
        }
        items = std::move(out);
    }

    // ---- Qwen3TTSSpeakerEncoder.sanitize (Qwen3TTSSpeakerEncoder.swift:324-354): the keys after the "speaker_encoder" component
    // (stripSpeakerEncoderPrefix); a 3-D ".weight" that fails checkArrayShapeQwen3 is taken for torch [out, in, k] and transposed to
    // [out, k, in].  Every other key is dropped.
    void sanitize_qwen3_speaker_encoder() {
        std::vector<WItem> out;
        for (auto& it : items) {
            std::vector<std::string> parts;                           // key.split(separator: "."): empty pieces dropped
            for (size_t a = 0; a <= it.name.size();) {
                const size_t b = std::min(it.name.find('.', a), it.name.size());
                if (b > a) parts.push_back(it.name.substr(a, b - a));
                a = b + 1;
            }
            std::string rest;
            for (size_t i = 0; i < parts.size(); ++i)
                if (parts[i] == "speaker_encoder") {
                    for (size_t j = i + 1; j < parts.size(); ++j) rest += (j > i + 1 ? "." : "") + parts[j];
                    break;
                }
            if (rest.empty()) continue;
            WItem t = it;
            t.name = rest;
            const bool weight = rest.size() >= 7 && rest.compare(rest.size() - 7, 7, ".weight") == 0;
            if (weight && t.ndim == 3 && !check_array_shape(t)) permute3(t, 0, 2, 1);
            out.push_back(std::move(t));
        }
        items = std::move(out);
    }

    // ---- Mimi.sanitize (Mimi/Mimi.swift:337-413), key for key: Swift's replacingOccurrences replaces every occurrence
    void sanitize_mimi() {
        auto replace_all = [](std::string& s, const std::string& from, const std::string& to) {
            for (size_t p = 0; (p = s.find(from, p)) != std::string::npos; p += to.size()) s.replace(p, from.size(), to);
        };
        auto ends_with = [](const std::string& s, const std::string& e) { return s.size() >= e.size() && s.compare(s.size() - e.size(), e.size(), e) == 0; };
        for (auto& t : items) {
            std::string k, seg;
            for (size_t a = 0;;) {                      // drop the leading "_" of every dot-separated segment
                const size_t b = t.name.find('.', a);
                seg = t.name.substr(a, b == std::string::npos ? std::string::npos : b - a);
                if (!seg.empty() && seg[0] == '_') seg = seg.substr(1);
                k += (a ? "." : "") + seg;
                if (b == std::string::npos) break;
                a = b + 1;
            }
            if (k.rfind("encoder.model.", 0) == 0) replace_all(k, "encoder.model.", "encoder.");
            if (k.rfind("decoder.model.", 0) == 0) replace_all(k, "decoder.model.", "decoder.");
            if (ends_with(k, ".in_proj_weight")) replace_all(k, ".in_proj_weight", ".in_proj.weight");
            if (ends_with(k, ".linear1.weight")) replace_all(k, ".linear1.weight", ".gating.linear1.weight");
            if (ends_with(k, ".linear2.weight")) replace_all(k, ".linear2.weight", ".gating.linear2.weight");
            const int dec_idx[4] = {2, 5, 8, 11}, enc_idx[4] = {1, 4, 7, 10};
            for (int l = 0; l < 4; ++l) {
                replace_all(k, "decoder." + std::to_string(dec_idx[l]) + ".", "decoder.layers." + std::to_string(l) + ".upsample.");
                replace_all(k, "decoder." + std::to_string(dec_idx[l] + 1) + ".", "decoder.layers." + std::to_string(l) + ".residuals.0.");
            }
            for (int l = 0; l < 4; ++l) {
                replace_all(k, "encoder." + std::to_string(enc_idx[l]) + ".", "encoder.layers." + std::to_string(l) + ".residuals.0.");
                replace_all(k, "encoder." + std::to_string(enc_idx[l] + 2) + ".", "encoder.layers." + std::to_string(l) + ".downsample.");
            }
            replace_all(k, "decoder.0.", "decoder.init_conv1d.");
            replace_all(k, "decoder.14.", "decoder.final_conv1d.");
            replace_all(k, "encoder.0.", "encoder.init_conv1d.");
            replace_all(k, "encoder.14.", "encoder.final_conv1d.");
            replace_all(k, ".block.1.", ".block.0.");
            replace_all(k, ".block.3.", ".block.1.");
            if ((ends_with(k, ".conv.weight") || ends_with(k, ".output_proj.weight") || ends_with(k, ".input_proj.weight")) && t.ndim >= 2) {
                if (t.ndim == 3) permute3(t, 0, 2, 1);
                else if (t.ndim == 2) {
                    const std::vector<float> v = as_f32(t);
                    const int64_t r = t.shape[0], c = t.shape[1];
                    auto o = std::make_shared<std::vector<uint8_t>>((size_t)(r * c) * 4);
                    float* of = (float*)o->data();
                    for (int64_t i = 0; i < r; ++i)
                        for (int64_t j = 0; j < c; ++j) of[j * r + i] = v[i * c + j];
                    t.owned = o; t.data = of; t.dtype = B2A_DTYPE_F32; t.shape[0] = c; t.shape[1] = r;
                } else {
                    throw Error(B2A_ERR_MODEL_NOT_INITIALIZED, "mimi sanitize: cannot swap the last axes of a 4-D tensor: " + t.name);
                }
            }
            if (ends_with(k, ".convtr.weight") && t.ndim == 3) {
                if (t.shape[1] == 1) permute3(t, 0, 2, 1);      // depthwise (C, 1, k) -> (C, k, 1)
                else permute3(t, 1, 2, 0);                      // (in, out, k) -> (out, k, in)
            }
            t.name = k;
        }
    }

    std::vector<b2a_tensor> table() const {
        std::vector<b2a_tensor> t(items.size());
        for (size_t i = 0; i < items.size(); ++i) {
            t[i].name = items[i].name.c_str(); t[i].dtype = items[i].dtype; t[i].ndim = items[i].ndim;
            for (int k = 0; k < 4; ++k) t[i].shape[k] = items[i].shape[k];
            t[i].data = items[i].data;
        }
        return t;
    }
};

extern "C" {

int32_t b2a_weights_load(const char* path, b2a_weights** out) {
    return guarded([&] {
        B2A_CHECK(out, B2A_ERR_INVALID_INPUT, "b2a_weights_load: null out");
        *out = nullptr;
        B2A_CHECK(path && *path, B2A_ERR_INVALID_INPUT, "b2a_weights_load: empty path");
        std::unique_ptr<b2a_weights> w(new b2a_weights());
        w->load(path);
        *out = w.release();
    });
}
int32_t b2a_weights_count(const b2a_weights* w) { return w ? (int32_t)w->items.size() : 0; }
int32_t b2a_weights_get(const b2a_weights* w, int32_t i, b2a_tensor* out) {
    return guarded([&] {
        B2A_CHECK(w && out && i >= 0 && i < (int32_t)w->items.size(), B2A_ERR_INVALID_INPUT, "b2a_weights_get: bad index");
        const WItem& it = w->items[i];
        out->name = it.name.c_str(); out->dtype = it.dtype; out->ndim = it.ndim;
        for (int k = 0; k < 4; ++k) out->shape[k] = it.shape[k];
        out->data = it.data;
    });
}
int32_t b2a_weights_sanitize_whisper(b2a_weights* w, int32_t* format) {
    return guarded([&] {
        B2A_CHECK(w, B2A_ERR_INVALID_INPUT, "b2a_weights_sanitize_whisper: null handle");
        const int f = w->sanitize_whisper();
        if (format) *format = f;
    });
}
int32_t b2a_weights_dequantize(b2a_weights* w, int32_t group_size, int32_t bits) {
    return guarded([&] {
        B2A_CHECK(w && bits > 0, B2A_ERR_INVALID_INPUT, "b2a_weights_dequantize: null handle or bits <= 0");
        QuantSpec q;
        q.group_size = group_size; q.bits = bits;
        w->dequantize_layers(q);
    });
}
// sanitize + de-quantise as config.json says, per-layer overrides included ("quantization": {group_size, bits, "<layer path>": false | {..}})
int32_t b2a_weights_sanitize_llama_config(b2a_weights* w, const char* config_path) {
    return guarded([&] {
        B2A_CHECK(w && config_path, B2A_ERR_INVALID_INPUT, "b2a_weights_sanitize_llama_config: null argument");
        const Json j = read_json_file(config_path);
        B2A_CHECK(j.kind == Json::Obj, B2A_ERR_MODEL_NOT_INITIALIZED, "config.json is not an object");
        w->sanitize_llama(j.number("tie_word_embeddings", 1) != 0, parse_quant(j));
    });
}
int32_t b2a_weights_sanitize_soprano_config(b2a_weights* w, const char* config_path) {
    return guarded([&] {
        B2A_CHECK(w && config_path, B2A_ERR_INVALID_INPUT, "b2a_weights_sanitize_soprano_config: null argument");
        const Json j = read_json_file(config_path);
        B2A_CHECK(j.kind == Json::Obj, B2A_ERR_MODEL_NOT_INITIALIZED, "config.json is not an object");
        w->sanitize_soprano(j.number("tie_word_embeddings", 0) != 0, parse_quant(j));
    });
}
int32_t b2a_weights_sanitize_llama(b2a_weights* w, int32_t tie_word_embeddings, int32_t group_size, int32_t bits) {
    return guarded([&] {
        B2A_CHECK(w, B2A_ERR_INVALID_INPUT, "b2a_weights_sanitize_llama: null handle");
        w->sanitize_llama(tie_word_embeddings != 0, group_size, bits);
    });
}
void b2a_weights_free(b2a_weights* w) { delete w; }

// config.json -> b2a_llama_config (LlamaTTSConfig.swift:100-166; rope_scaling defaults LlamaTTS.swift:114-118) and the quantisation block
int32_t b2a_tts_config_from_json(const char* config_path, int32_t max_batch, int32_t max_context, b2a_llama_config* cfg,
                                 int32_t* quant_group_size, int32_t* quant_bits) {
    return guarded([&] {
        B2A_CHECK(config_path && cfg, B2A_ERR_INVALID_INPUT, "b2a_tts_config_from_json: null argument");
        const Json j = read_json_file(config_path);
        B2A_CHECK(j.kind == Json::Obj, B2A_ERR_MODEL_NOT_INITIALIZED, "config.json is not an object");
        for (const char* k : {"hidden_size", "num_hidden_layers", "intermediate_size", "num_attention_heads", "rms_norm_eps", "vocab_size"})
            B2A_CHECK(j.has(k), B2A_ERR_MODEL_NOT_INITIALIZED, std::string("config.json: missing ") + k);      // non-optional decode()s
        b2a_llama_config c{};
        c.hidden_size = (int)j.number("hidden_size", 0); c.num_hidden_layers = (int)j.number("num_hidden_layers", 0);
        c.intermediate_size = (int)j.number("intermediate_size", 0); c.num_attention_heads = (int)j.number("num_attention_heads", 0);
        c.num_key_value_heads = (int)j.number("num_key_value_heads", c.num_attention_heads);
        c.head_dim = (int)j.number("head_dim", c.num_attention_heads ? c.hidden_size / c.num_attention_heads : 0);
        c.vocab_size = (int)j.number("vocab_size", 0);
        c.rms_norm_eps = (float)j.number("rms_norm_eps", 1e-5); c.rope_theta = (float)j.number("rope_theta", 10000.0);   // LlamaTTSConfig.swift:25
        c.tie_word_embeddings = (int)j.number("tie_word_embeddings", 1);
        // decoded by the reference but with no code path here: reject instead of silently computing something else
        B2A_CHECK(j.number("rope_traditional", 0) == 0, B2A_ERR_INVALID_INPUT, "config.json: rope_traditional = true is not supported");
        B2A_CHECK(j.number("attention_bias", 0) == 0 && j.number("mlp_bias", 0) == 0, B2A_ERR_INVALID_INPUT,
                  "config.json: attention_bias / mlp_bias = true are not supported");
        c.rope_factor = 32.f; c.rope_low_freq_factor = 1.f; c.rope_high_freq_factor = 4.f; c.rope_old_context_len = 8192.f;
        if (const Json* rs = j.find("rope_scaling"); rs && rs->kind == Json::Obj) {
            B2A_CHECK(rs->has("factor"), B2A_ERR_MODEL_NOT_INITIALIZED, "rope_scaling must contain 'factor'");
            B2A_CHECK(rs->has("type") || rs->has("rope_type"), B2A_ERR_MODEL_NOT_INITIALIZED, "rope_scaling must contain either 'type' or 'rope_type'");
            c.rope_factor = (float)rs->number("factor", 32.0);
            c.rope_low_freq_factor = (float)rs->number("low_freq_factor", 1.0);
            c.rope_high_freq_factor = (float)rs->number("high_freq_factor", 4.0);
            c.rope_old_context_len = (float)rs->number("original_max_position_embeddings", 8192.0);
        }
        c.max_batch = max_batch; c.max_context = max_context;
        *cfg = c;
        int gs = 0, bits = 0;
        if (const Json* q = j.find("quantization"); q && q->kind == Json::Obj) { gs = (int)q->number("group_size", 64); bits = (int)q->number("bits", 4); }
        if (quant_group_size) *quant_group_size = gs;
        if (quant_bits) *quant_bits = bits;
    });
}

// LlamaTTSModel.fromModelDirectory (LlamaTTS.swift:942-977): config.json + every *.safetensors -> sanitize -> (de)quantise -> create.
int32_t b2a_tts_create_from_directory(const char* model_dir, int32_t device, int32_t max_batch, int32_t max_context, b2a_snac* snac,
                                      b2a_tts** out) {
    return guarded([&] {
        B2A_CHECK(model_dir && out, B2A_ERR_INVALID_INPUT, "b2a_tts_create_from_directory: null argument");
        *out = nullptr;
        b2a_llama_config cfg{};
        int gs = 0, bits = 0;
        const std::string dir = model_dir;
        int32_t st = b2a_tts_config_from_json((dir + "/config.json").c_str(), max_batch, max_context, &cfg, &gs, &bits);
        if (st != B2A_OK) throw Error(st, b2a_last_error());
        std::unique_ptr<b2a_weights> w(new b2a_weights());
        w->load(dir);
        w->sanitize_llama(cfg.tie_word_embeddings != 0, parse_quant(read_json_file(dir + "/config.json")));
        const std::vector<b2a_tensor> tab = w->table();
        st = b2a_tts_create(device, &cfg, tab.data(), (int32_t)tab.size(), snac, out);
        if (st != B2A_OK) throw Error(st, b2a_last_error());
    });
}

// config.json -> b2a_qwen3_lm_config (Qwen3Configuration.init(from:), Config.swift:50-73): the eight decode()d keys are required, the rest
// take the reference's defaults; rope_scaling counts only as {"type": "linear", "factor": f} (Qwen3Attention, Qwen3.swift:177-188)
int32_t b2a_qwen3_lm_config_from_json(const char* config_path, int32_t max_batch, int32_t max_context, b2a_qwen3_lm_config* cfg,
                                      int32_t* quant_group_size, int32_t* quant_bits) {
    return guarded([&] {
        B2A_CHECK(config_path && cfg, B2A_ERR_INVALID_INPUT, "b2a_qwen3_lm_config_from_json: null argument");
        const Json j = read_json_file(config_path);
        B2A_CHECK(j.kind == Json::Obj, B2A_ERR_MODEL_NOT_INITIALIZED, "config.json is not an object");
        for (const char* k : {"hidden_size", "num_hidden_layers", "intermediate_size", "num_attention_heads", "rms_norm_eps", "vocab_size",
                              "num_key_value_heads", "head_dim"})
            B2A_CHECK(j.has(k), B2A_ERR_MODEL_NOT_INITIALIZED, std::string("config.json: missing ") + k);
        b2a_qwen3_lm_config c{};
        c.hidden_size = (int)j.number("hidden_size", 0); c.num_hidden_layers = (int)j.number("num_hidden_layers", 0);
        c.intermediate_size = (int)j.number("intermediate_size", 0); c.num_attention_heads = (int)j.number("num_attention_heads", 0);
        c.num_key_value_heads = (int)j.number("num_key_value_heads", 0); c.head_dim = (int)j.number("head_dim", 0);
        c.vocab_size = (int)j.number("vocab_size", 0); c.rms_norm_eps = (float)j.number("rms_norm_eps", 0.0);
        c.rope_theta = (float)j.number("rope_theta", 1000000.0);
        c.rope_linear_factor = 1.f;
        if (const Json* rs = j.find("rope_scaling"); rs && rs->kind == Json::Obj) {
            const Json* ty = rs->find("type");
            if (ty && ty->kind == Json::Str && ty->str == "linear" && rs->has("factor")) {
                const Json* f = rs->find("factor");
                B2A_CHECK(f->kind == Json::Num && f->num > 0, B2A_ERR_MODEL_NOT_INITIALIZED, "rope_scaling.factor must be a positive number");
                c.rope_linear_factor = (float)f->num;
            }
        }
        c.tie_word_embeddings = (int)j.number("tie_word_embeddings", 0);
        c.max_position_embeddings = (int)j.number("max_position_embeddings", 32768);
        c.sample_rate = (int)j.number("sample_rate", 24000);
        c.eos_token_id = (int)j.number("eos_token_id", 151645);
        c.max_batch = max_batch; c.max_context = max_context;
        *cfg = c;
        int gs = 0, bits = 0;
        if (const Json* q = j.find("quantization"); q && q->kind == Json::Obj) { gs = (int)q->number("group_size", 64); bits = (int)q->number("bits", 4); }
        if (quant_group_size) *quant_group_size = gs;
        if (quant_bits) *quant_bits = bits;
    });
}

// Qwen3Model.fromModelDirectory (Qwen3.swift:892-930): config.json + every *.safetensors -> sanitize -> (de)quantise -> create
int32_t b2a_qwen3_lm_create_from_directory(const char* model_dir, int32_t device, int32_t max_batch, int32_t max_context, b2a_snac* snac,
                                           b2a_tts** out) {
    return guarded([&] {
        B2A_CHECK(model_dir && out, B2A_ERR_INVALID_INPUT, "b2a_qwen3_lm_create_from_directory: null argument");
        *out = nullptr;
        b2a_qwen3_lm_config cfg{};
        const std::string dir = model_dir;
        int32_t st = b2a_qwen3_lm_config_from_json((dir + "/config.json").c_str(), max_batch, max_context, &cfg, nullptr, nullptr);
        if (st != B2A_OK) throw Error(st, b2a_last_error());
        std::unique_ptr<b2a_weights> w(new b2a_weights());
        w->load(dir);
        w->sanitize_llama(cfg.tie_word_embeddings != 0, parse_quant(read_json_file(dir + "/config.json")));
        const std::vector<b2a_tensor> tab = w->table();
        st = b2a_qwen3_lm_create(device, &cfg, tab.data(), (int32_t)tab.size(), snac, out);
        if (st != B2A_OK) throw Error(st, b2a_last_error());
    });
}

// config.json -> b2a_soprano_config (SopranoConfiguration.init(from:), SopranoConfig.swift:133-175): the seven decode()d keys are required,
// the rest take the reference's defaults; then fromModelDirectory's decoder rule (Soprano.swift:934-941) on the repo name
static std::string lower(std::string s) {
    for (auto& ch : s) ch = (char)std::tolower((unsigned char)ch);
    return s;
}
static std::string base_name(std::string p) {
    while (p.size() > 1 && p.back() == '/') p.pop_back();
    const size_t i = p.rfind('/');
    return i == std::string::npos ? p : p.substr(i + 1);
}
int32_t b2a_soprano_config_from_json(const char* config_path, const char* repo_hint, int32_t max_batch, int32_t max_context,
                                     b2a_soprano_config* cfg, int32_t* quant_group_size, int32_t* quant_bits) {
    return guarded([&] {
        B2A_CHECK(config_path && cfg, B2A_ERR_INVALID_INPUT, "b2a_soprano_config_from_json: null argument");
        const Json j = read_json_file(config_path);
        B2A_CHECK(j.kind == Json::Obj, B2A_ERR_MODEL_NOT_INITIALIZED, "config.json is not an object");
        for (const char* k : {"hidden_size", "num_hidden_layers", "intermediate_size", "num_attention_heads", "num_key_value_heads", "head_dim",
                              "vocab_size"})
            B2A_CHECK(j.has(k), B2A_ERR_MODEL_NOT_INITIALIZED, std::string("config.json: missing ") + k);
        b2a_soprano_config c{};
        c.hidden_size = (int)j.number("hidden_size", 0); c.num_hidden_layers = (int)j.number("num_hidden_layers", 0);
        c.intermediate_size = (int)j.number("intermediate_size", 0); c.num_attention_heads = (int)j.number("num_attention_heads", 0);
        c.num_key_value_heads = (int)j.number("num_key_value_heads", 0); c.head_dim = (int)j.number("head_dim", 0);
        c.vocab_size = (int)j.number("vocab_size", 0);
        c.max_position_embeddings = (int)j.number("max_position_embeddings", 512);
        c.rms_norm_eps = (float)j.number("rms_norm_eps", 1e-6); c.rope_theta = (float)j.number("rope_theta", 10000.0);
        c.tie_word_embeddings = (int)j.number("tie_word_embeddings", 0);
        c.bos_token_id = (int)j.number("bos_token_id", 1); c.eos_token_id = (int)j.number("eos_token_id", 2);
        c.pad_token_id = (int)j.number("pad_token_id", 0); c.stop_token_id = 3;
        c.sample_rate = (int)j.number("sample_rate", 32000);
        c.decoder_num_layers = (int)j.number("decoder_num_layers", 8); c.decoder_dim = (int)j.number("decoder_dim", 768);
        c.decoder_intermediate_dim = (int)j.number("decoder_intermediate_dim", 2304); c.hop_length = (int)j.number("hop_length", 512);
        c.n_fft = (int)j.number("n_fft", 2048); c.upscale = (int)j.number("upscale", 4); c.input_kernel = (int)j.number("input_kernel", 1);
        c.dw_kernel = (int)j.number("dw_kernel", 3); c.token_size = (int)j.number("token_size", 2048);
        c.receptive_field = (int)j.number("receptive_field", 4);
        std::string cp = config_path;
        const size_t sl = cp.rfind('/');
        const std::string repo = repo_hint ? std::string(repo_hint) : base_name(sl == std::string::npos ? std::string(".") : cp.substr(0, sl));
        if (lower(repo).find("soprano-1.1") == std::string::npos) {      // the older decoder, whatever config.json says
            c.decoder_dim = 512; c.decoder_intermediate_dim = 1536; c.input_kernel = 3;
        }
        c.max_batch = max_batch; c.max_context = max_context;
        *cfg = c;
        int gs = 0, bits = 0;
        if (const Json* q = j.find("quantization"); q && q->kind == Json::Obj) { gs = (int)q->number("group_size", 64); bits = (int)q->number("bits", 4); }
        if (quant_group_size) *quant_group_size = gs;
        if (quant_bits) *quant_bits = bits;
    });
}

// model.stopTokenId = tokenizer.eosTokenId ?? 3 (Soprano.swift:971-973): tokenizer_config.json's eos_token resolved through tokenizer.json's
// added_tokens or model.vocab; 3 when either file or the token is missing
static int soprano_stop_token(const std::string& dir) {
    struct stat st{};
    if (stat((dir + "/tokenizer_config.json").c_str(), &st) != 0 || stat((dir + "/tokenizer.json").c_str(), &st) != 0) return 3;
    const Json tc = read_json_file(dir + "/tokenizer_config.json");
    const Json* e = tc.find("eos_token");
    std::string eos;
    if (e && e->kind == Json::Str) eos = e->str;
    else if (e && e->kind == Json::Obj && e->find("content") && e->find("content")->kind == Json::Str) eos = e->find("content")->str;
    if (eos.empty()) return 3;
    const Json tj = read_json_file(dir + "/tokenizer.json");
    if (const Json* at = tj.find("added_tokens"); at && at->kind == Json::Arr)
        for (const Json& t : at->arr) {
            const Json* c = t.find("content");
            if (c && c->kind == Json::Str && c->str == eos && t.has("id")) return (int)t.number("id", 3);
        }
    if (const Json* m = tj.find("model"); m && m->kind == Json::Obj)
        if (const Json* v = m->find("vocab"); v && v->kind == Json::Obj)
            if (const Json* id = v->find(eos); id && id->kind == Json::Num) return (int)id->num;
    return 3;
}

int32_t b2a_soprano_create_from_directory(const char* model_dir, const char* repo_hint, int32_t device, int32_t max_batch,
                                          int32_t max_context, b2a_tts** out) {
    return guarded([&] {
        B2A_CHECK(model_dir && out, B2A_ERR_INVALID_INPUT, "b2a_soprano_create_from_directory: null argument");
        *out = nullptr;
        b2a_soprano_config cfg{};
        const std::string dir = model_dir;
        const std::string repo = repo_hint ? std::string(repo_hint) : base_name(dir);
        int32_t st = b2a_soprano_config_from_json((dir + "/config.json").c_str(), repo.c_str(), max_batch, max_context, &cfg, nullptr, nullptr);
        if (st != B2A_OK) throw Error(st, b2a_last_error());
        cfg.stop_token_id = soprano_stop_token(dir);
        std::unique_ptr<b2a_weights> w(new b2a_weights());
        w->load(dir);
        w->sanitize_soprano(cfg.tie_word_embeddings != 0, parse_quant(read_json_file(dir + "/config.json")));
        const std::vector<b2a_tensor> tab = w->table();
        st = b2a_soprano_create(device, &cfg, tab.data(), (int32_t)tab.size(), out);
        if (st != B2A_OK) throw Error(st, b2a_last_error());
    });
}

// config.json -> b2a_qwen3_talker_config: "talker_config" with its nested "code_predictor_config" (Qwen3TTSConfig.swift:45-63,268-292; the
// same defaults), max_batch / max_context from the caller.
static b2a_qwen3_talker_config qwen3_talker_config_of(const Json& root, int max_batch, int max_context) {
    Json empty;
    empty.kind = Json::Obj;
    const Json* tj = root.find("talker_config");
    const Json& t = (tj && tj->kind == Json::Obj) ? *tj : empty;
    const Json* pj = t.find("code_predictor_config");
    const Json& p = (pj && pj->kind == Json::Obj) ? *pj : empty;
    b2a_qwen3_talker_config c{};
    c.vocab_size = (int)t.number("vocab_size", 3072); c.hidden_size = (int)t.number("hidden_size", 1024);
    c.intermediate_size = (int)t.number("intermediate_size", 3072); c.num_hidden_layers = (int)t.number("num_hidden_layers", 28);
    c.num_attention_heads = (int)t.number("num_attention_heads", 16); c.num_key_value_heads = (int)t.number("num_key_value_heads", 8);
    c.head_dim = (int)t.number("head_dim", 128); c.rms_norm_eps = (float)t.number("rms_norm_eps", 1e-6);
    c.rope_theta = (float)t.number("rope_theta", 1000000.0); c.num_code_groups = (int)t.number("num_code_groups", 16);
    c.text_hidden_size = (int)t.number("text_hidden_size", 2048); c.text_vocab_size = (int)t.number("text_vocab_size", 151936);
    c.codec_eos_token_id = (int)t.number("codec_eos_token_id", 2150);
    c.cp_vocab_size = (int)p.number("vocab_size", 2048); c.cp_hidden_size = (int)p.number("hidden_size", 1024);
    c.cp_intermediate_size = (int)p.number("intermediate_size", 3072); c.cp_num_hidden_layers = (int)p.number("num_hidden_layers", 5);
    c.cp_num_attention_heads = (int)p.number("num_attention_heads", 16); c.cp_num_key_value_heads = (int)p.number("num_key_value_heads", 8);
    c.cp_head_dim = (int)p.number("head_dim", 128); c.cp_rms_norm_eps = (float)p.number("rms_norm_eps", 1e-6);
    c.cp_rope_theta = (float)p.number("rope_theta", 1000000.0);
    B2A_CHECK(t.number("attention_bias", 0) == 0 && p.number("attention_bias", 0) == 0, B2A_ERR_INVALID_INPUT,
              "qwen3 talker: attention_bias = true is not supported");
    c.max_batch = max_batch; c.max_context = max_context;
    return c;
}

int32_t b2a_qwen3_talker_config_from_json(const char* config_path, int32_t max_batch, int32_t max_context, b2a_qwen3_talker_config* cfg) {
    return guarded([&] {
        B2A_CHECK(config_path && cfg, B2A_ERR_INVALID_INPUT, "b2a_qwen3_talker_config_from_json: null argument");
        const Json j = read_json_file(config_path);
        B2A_CHECK(j.kind == Json::Obj, B2A_ERR_MODEL_NOT_INITIALIZED, "config.json is not an object");
        *cfg = qwen3_talker_config_of(j, max_batch, max_context);
    });
}

int32_t b2a_weights_sanitize_qwen3_talker(b2a_weights* w, const char* config_path) {
    return guarded([&] {
        B2A_CHECK(w, B2A_ERR_INVALID_INPUT, "b2a_weights_sanitize_qwen3_talker: null handle");
        QuantSpec q;
        if (config_path && *config_path) q = parse_quant(read_json_file(config_path));
        w->sanitize_qwen3_talker(q);
    });
}

// Qwen3TTSModel.fromModelDirectory (Qwen3TTS.swift:1136-1175), the talker half: config.json + every *.safetensors -> sanitize ->
// (de)quantise -> create.  The tokenizer, the speaker encoder and the speech tokenizer (b2a_speech_tokenizer_create_from_directory on
// <dir>/speech_tokenizer) are the caller's.
int32_t b2a_qwen3_talker_create_from_directory(const char* model_dir, int32_t device, int32_t max_batch, int32_t max_context,
                                               b2a_qwen3_talker** out) {
    return guarded([&] {
        B2A_CHECK(model_dir && out, B2A_ERR_INVALID_INPUT, "b2a_qwen3_talker_create_from_directory: null argument");
        *out = nullptr;
        const std::string dir = model_dir;
        const Json j = read_json_file(dir + "/config.json");
        B2A_CHECK(j.kind == Json::Obj, B2A_ERR_MODEL_NOT_INITIALIZED, "config.json is not an object");
        const b2a_qwen3_talker_config cfg = qwen3_talker_config_of(j, max_batch, max_context);
        std::unique_ptr<b2a_weights> w(new b2a_weights());
        w->load(dir);
        w->sanitize_qwen3_talker(parse_quant(j));
        const std::vector<b2a_tensor> tab = w->table();
        const int32_t st = b2a_qwen3_talker_create(device, &cfg, tab.data(), (int32_t)tab.size(), out);
        if (st != B2A_OK) throw Error(st, b2a_last_error());
    });
}

int32_t b2a_weights_sanitize_speech_tokenizer(b2a_weights* w) {
    return guarded([&] {
        B2A_CHECK(w, B2A_ERR_INVALID_INPUT, "b2a_weights_sanitize_speech_tokenizer: null handle");
        w->sanitize_speech_tokenizer();
    });
}

// speech_tokenizer/config.json -> b2a_speech_tokenizer_config (Qwen3TTSTokenizerConfig / ...DecoderConfig, Qwen3TTSConfig.swift:358-385,518-527).
// A missing file means "all defaults", as loadSpeechTokenizer does (Qwen3TTS.swift:1246-1255).
int32_t b2a_speech_tokenizer_config_from_json(const char* config_path, int32_t max_batch, int32_t max_cache_frames, b2a_speech_tokenizer_config* cfg,
                                              int32_t* decode_upsample_rate) {
    return guarded([&] {
        B2A_CHECK(cfg, B2A_ERR_INVALID_INPUT, "b2a_speech_tokenizer_config_from_json: null argument");
        Json j;
        j.kind = Json::Obj;
        struct stat st{};
        if (config_path && *config_path && stat(config_path, &st) == 0) j = read_json_file(config_path);
        B2A_CHECK(j.kind == Json::Obj, B2A_ERR_MODEL_NOT_INITIALIZED, "speech tokenizer config.json is not an object");
        Json empty;
        empty.kind = Json::Obj;
        const Json* dj = j.find("decoder_config");
        const Json& d = (dj && dj->kind == Json::Obj) ? *dj : empty;
        b2a_speech_tokenizer_config c{};
        c.codebook_size = (int)d.number("codebook_size", 2048); c.codebook_dim = (int)d.number("codebook_dim", 512);
        c.latent_dim = (int)d.number("latent_dim", 1024); c.decoder_dim = (int)d.number("decoder_dim", 1536);
        c.hidden_size = (int)d.number("hidden_size", 512); c.intermediate_size = (int)d.number("intermediate_size", 1024);
        c.head_dim = (int)d.number("head_dim", 64); c.num_attention_heads = (int)d.number("num_attention_heads", 16);
        c.num_key_value_heads = (int)d.number("num_key_value_heads", 16); c.num_hidden_layers = (int)d.number("num_hidden_layers", 8);
        c.num_quantizers = (int)d.number("num_quantizers", 16); c.num_semantic_quantizers = (int)d.number("num_semantic_quantizers", 1);
        c.rms_norm_eps = (float)d.number("rms_norm_eps", 1e-5); c.rope_theta = (float)d.number("rope_theta", 10000.0);
        c.attention_bias = (int)d.number("attention_bias", 0);
        auto list = [&](const char* key, std::initializer_list<int> dflt, int32_t* dst, int32_t* n) {
            std::vector<int> v(dflt);
            if (const Json* a = d.find(key); a && a->kind == Json::Arr) { v.clear(); for (auto& e : a->arr) v.push_back((int)e.num); }
            B2A_CHECK(v.size() <= 8, B2A_ERR_MODEL_NOT_INITIALIZED, std::string("speech tokenizer config: more than 8 entries in ") + key);
            *n = (int32_t)v.size();
            for (size_t i = 0; i < v.size(); ++i) dst[i] = v[i];
        };
        list("upsample_rates", {8, 5, 4, 3}, c.upsample_rates, &c.num_upsample_rates);
        list("upsampling_ratios", {2, 2}, c.upsampling_ratios, &c.num_upsampling_ratios);
        c.max_batch = max_batch; c.max_cache_frames = max_cache_frames;
        *cfg = c;
        if (decode_upsample_rate) *decode_upsample_rate = (int32_t)j.number("decode_upsample_rate", 1920);
    });
}

// loadSpeechTokenizer (Qwen3TTS.swift:1244-1275): <dir>/config.json (optional) + every *.safetensors -> sanitize -> create.
int32_t b2a_speech_tokenizer_create_from_directory(const char* dir, int32_t device, int32_t max_batch, int32_t max_cache_frames,
                                                   b2a_speech_tokenizer** out, int32_t* decode_upsample_rate) {
    return guarded([&] {
        B2A_CHECK(dir && out, B2A_ERR_INVALID_INPUT, "b2a_speech_tokenizer_create_from_directory: null argument");
        *out = nullptr;
        b2a_speech_tokenizer_config cfg{};
        const std::string d = dir;
        int32_t st = b2a_speech_tokenizer_config_from_json((d + "/config.json").c_str(), max_batch, max_cache_frames, &cfg, decode_upsample_rate);
        if (st != B2A_OK) throw Error(st, b2a_last_error());
        std::unique_ptr<b2a_weights> w(new b2a_weights());
        w->load(d);
        w->sanitize_speech_tokenizer();
        const std::vector<b2a_tensor> tab = w->table();
        st = b2a_speech_tokenizer_create(device, &cfg, tab.data(), (int32_t)tab.size(), out);
        if (st != B2A_OK) throw Error(st, b2a_last_error());
    });
}

int32_t b2a_weights_sanitize_speech_tokenizer_encoder(b2a_weights* w) {
    return guarded([&] {
        B2A_CHECK(w, B2A_ERR_INVALID_INPUT, "b2a_weights_sanitize_speech_tokenizer_encoder: null handle");
        w->sanitize_speech_tokenizer_encoder();
    });
}

// speech_tokenizer/config.json's "encoder_config" (Qwen3TTSTokenizerEncoderConfig, Qwen3TTSConfig.swift:391-494, the same defaults) and
// "encoder_valid_num_quantizers" (:518-527, default 16).  No file or no block is the reference's encoderConfig == nil: no encoder.
int32_t b2a_speech_tokenizer_encoder_config_from_json(const char* config_path, b2a_speech_tokenizer_encoder_config* cfg) {
    return guarded([&] {
        B2A_CHECK(config_path && cfg, B2A_ERR_INVALID_INPUT, "b2a_speech_tokenizer_encoder_config_from_json: null argument");
        struct stat st{};
        B2A_CHECK(stat(config_path, &st) == 0, B2A_ERR_MODEL_NOT_INITIALIZED, "speech tokenizer: no config.json, so no encoder_config");
        const Json j = read_json_file(config_path);
        B2A_CHECK(j.kind == Json::Obj, B2A_ERR_MODEL_NOT_INITIALIZED, "speech tokenizer config.json is not an object");
        const Json* ej = j.find("encoder_config");
        B2A_CHECK(ej && ej->kind == Json::Obj, B2A_ERR_MODEL_NOT_INITIALIZED, "speech tokenizer config.json has no encoder_config");
        const Json& e = *ej;
        b2a_speech_tokenizer_encoder_config c{};
        c.sampling_rate = (int)e.number("sampling_rate", 24000); c.frame_rate = (float)e.number("frame_rate", 12.5);
        c.audio_channels = (int)e.number("audio_channels", 1); c.num_filters = (int)e.number("num_filters", 64);
        c.num_residual_layers = (int)e.number("num_residual_layers", 1);
        std::vector<int> ratios = {8, 6, 5, 4};
        if (const Json* a = e.find("upsampling_ratios"); a && a->kind == Json::Arr) { ratios.clear(); for (auto& x : a->arr) ratios.push_back((int)x.num); }
        B2A_CHECK(ratios.size() <= 8, B2A_ERR_MODEL_NOT_INITIALIZED, "speech tokenizer encoder config: more than 8 upsampling_ratios");
        c.num_upsampling_ratios = (int32_t)ratios.size();
        for (size_t i = 0; i < ratios.size(); ++i) c.upsampling_ratios[i] = ratios[i];
        c.kernel_size = (int)e.number("kernel_size", 7); c.residual_kernel_size = (int)e.number("residual_kernel_size", 3);
        c.last_kernel_size = (int)e.number("last_kernel_size", 3); c.compress = (int)e.number("compress", 2);
        c.use_causal_conv = (int)e.number("use_causal_conv", 1); c.use_conv_shortcut = (int)e.number("use_conv_shortcut", 0);
        c.hidden_size = (int)e.number("hidden_size", 512); c.intermediate_size = (int)e.number("intermediate_size", 2048);
        c.num_hidden_layers = (int)e.number("num_hidden_layers", 8); c.num_attention_heads = (int)e.number("num_attention_heads", 8);
        c.num_key_value_heads = (int)e.number("num_key_value_heads", 8);
        c.head_dim = c.num_attention_heads > 0 ? c.hidden_size / c.num_attention_heads : 0;     // the transformer's dModel / numHeads
        c.rope_theta = (float)e.number("rope_theta", 10000.0);
        c.codebook_size = (int)e.number("codebook_size", 2048); c.codebook_dim = (int)e.number("codebook_dim", 256);
        c.num_quantizers = (int)e.number("num_quantizers", 32);
        c.valid_num_quantizers = (int)j.number("encoder_valid_num_quantizers", 16);
        *cfg = c;
    });
}

// the encoder half of loadSpeechTokenizer (Qwen3TTS.swift:1244-1275): <dir>/config.json + every *.safetensors -> sanitize -> create
int32_t b2a_speech_tokenizer_encoder_create_from_directory(const char* dir, int32_t device, b2a_speech_tokenizer_encoder** out) {
    return guarded([&] {
        B2A_CHECK(dir && out, B2A_ERR_INVALID_INPUT, "b2a_speech_tokenizer_encoder_create_from_directory: null argument");
        *out = nullptr;
        b2a_speech_tokenizer_encoder_config cfg{};
        const std::string d = dir;
        int32_t st = b2a_speech_tokenizer_encoder_config_from_json((d + "/config.json").c_str(), &cfg);
        if (st != B2A_OK) throw Error(st, b2a_last_error());
        std::unique_ptr<b2a_weights> w(new b2a_weights());
        w->load(d);
        w->sanitize_speech_tokenizer_encoder();
        B2A_CHECK(!w->items.empty(), B2A_ERR_MODEL_NOT_INITIALIZED, "speech tokenizer: the checkpoint has no encoder weights");
        const std::vector<b2a_tensor> tab = w->table();
        st = b2a_speech_tokenizer_encoder_create(device, &cfg, tab.data(), (int32_t)tab.size(), out);
        if (st != B2A_OK) throw Error(st, b2a_last_error());
    });
}

int32_t b2a_weights_sanitize_qwen3_speaker_encoder(b2a_weights* w) {
    return guarded([&] {
        B2A_CHECK(w, B2A_ERR_INVALID_INPUT, "b2a_weights_sanitize_qwen3_speaker_encoder: null handle");
        w->sanitize_qwen3_speaker_encoder();
    });
}

// config.json's "speaker_encoder_config" (Qwen3TTSSpeakerEncoderConfig, Qwen3TTSConfig.swift:92-103: the same keys and defaults; a
// missing block is all defaults, as decodeIfPresent gives).  The three lists must have the same length, at most 8.
static b2a_qwen3_speaker_encoder_config qwen3_speaker_config_of(const Json& root) {
    Json empty;
    empty.kind = Json::Obj;
    const Json* sj = root.find("speaker_encoder_config");
    const Json& e = (sj && sj->kind == Json::Obj) ? *sj : empty;
    b2a_qwen3_speaker_encoder_config c{};
    c.mel_dim = (int)e.number("mel_dim", 128); c.enc_dim = (int)e.number("enc_dim", 1024);
    c.enc_attention_channels = (int)e.number("enc_attention_channels", 128); c.enc_res2net_scale = (int)e.number("enc_res2net_scale", 8);
    c.enc_se_channels = (int)e.number("enc_se_channels", 128); c.sample_rate = (int)e.number("sample_rate", 24000);
    auto list = [&](const char* key, std::initializer_list<int> dflt, int32_t* dst) {
        std::vector<int> v(dflt);
        if (const Json* a = e.find(key); a && a->kind == Json::Arr) { v.clear(); for (auto& x : a->arr) v.push_back((int)x.num); }
        B2A_CHECK(v.size() <= 8, B2A_ERR_INVALID_INPUT, std::string("speaker encoder config: more than 8 entries in ") + key);
        for (size_t i = 0; i < v.size(); ++i) dst[i] = v[i];
        return (int)v.size();
    };
    const int n0 = list("enc_channels", {512, 512, 512, 512, 1536}, c.enc_channels);
    const int n1 = list("enc_kernel_sizes", {5, 3, 3, 3, 1}, c.enc_kernel_sizes);
    const int n2 = list("enc_dilations", {1, 2, 3, 4, 1}, c.enc_dilations);
    B2A_CHECK(n0 == n1 && n0 == n2, B2A_ERR_INVALID_INPUT, "speaker encoder config: enc_channels, enc_kernel_sizes and enc_dilations must have the same length");
    c.num_enc_layers = n0;
    return c;
}

int32_t b2a_qwen3_speaker_encoder_config_from_json(const char* config_path, b2a_qwen3_speaker_encoder_config* cfg) {
    return guarded([&] {
        B2A_CHECK(config_path && cfg, B2A_ERR_INVALID_INPUT, "b2a_qwen3_speaker_encoder_config_from_json: null argument");
        const Json j = read_json_file(config_path);
        B2A_CHECK(j.kind == Json::Obj, B2A_ERR_MODEL_NOT_INITIALIZED, "config.json is not an object");
        *cfg = qwen3_speaker_config_of(j);
    });
}

// The speaker-encoder half of Qwen3TTSModel.fromModelDirectory (Qwen3TTS.swift:46-48, 1224-1237): only a "base" checkpoint builds
// the encoder; config.json + every *.safetensors -> sanitize -> create.
int32_t b2a_qwen3_speaker_encoder_create_from_directory(const char* model_dir, int32_t device, b2a_qwen3_speaker_encoder** out) {
    return guarded([&] {
        B2A_CHECK(model_dir && out, B2A_ERR_INVALID_INPUT, "b2a_qwen3_speaker_encoder_create_from_directory: null argument");
        *out = nullptr;
        const std::string dir = model_dir;
        const Json j = read_json_file(dir + "/config.json");
        B2A_CHECK(j.kind == Json::Obj, B2A_ERR_MODEL_NOT_INITIALIZED, "config.json is not an object");
        const Json* mt = j.find("tts_model_type");
        B2A_CHECK(mt && mt->kind == Json::Str && mt->str == "base", B2A_ERR_MODEL_NOT_INITIALIZED,
                  "speaker encoder: only a Base checkpoint (tts_model_type \"base\") has one");
        const b2a_qwen3_speaker_encoder_config cfg = qwen3_speaker_config_of(j);
        std::unique_ptr<b2a_weights> w(new b2a_weights());
        w->load(dir);
        w->sanitize_qwen3_speaker_encoder();
        B2A_CHECK(!w->items.empty(), B2A_ERR_MODEL_NOT_INITIALIZED, "speaker encoder: the checkpoint has no speaker_encoder weights");
        const std::vector<b2a_tensor> tab = w->table();
        const int32_t st = b2a_qwen3_speaker_encoder_create(device, &cfg, tab.data(), (int32_t)tab.size(), out);
        if (st != B2A_OK) throw Error(st, b2a_last_error());
    });
}

// ---- the other two host helpers of DSP.swift (not on the mel path; the reference's own tests hold known answers for them)
// hammingWindow (Sources/MLXAudioCore/DSP.swift:25-42): periodic = the first `size` points of the (size + 1)-point window
int32_t b2a_hamming_window(int32_t size, int32_t periodic, float* out) {
    return guarded([&] {
        B2A_CHECK(size >= 0 && (out || size == 0), B2A_ERR_INVALID_INPUT, "b2a_hamming_window: bad arguments");
        if (size == 0) return;
        if (size == 1) { out[0] = 1.0f; return; }
        const int eff = periodic ? size + 1 : size;
        const float denom = (float)(eff - 1);
        for (int n = 0; n < size; ++n) out[n] = 0.54f - 0.46f * cosf(2.0f * (float)M_PI * (float)n / denom);
    });
}
// powerToDB (DSP.swift:61-73): 10 log10(max(x, amin)), then max(., global max - top_db) when top_db >= 0
int32_t b2a_power_to_db(const float* spectrogram, int64_t n, float amin, float top_db, float* out) {
    return guarded([&] {
        B2A_CHECK(n >= 0 && (n == 0 || (spectrogram && out)), B2A_ERR_INVALID_INPUT, "b2a_power_to_db: bad arguments");
        float mx = -INFINITY;
        for (int64_t i = 0; i < n; ++i) { out[i] = 10.0f * log10f(std::max(spectrogram[i], amin)); mx = std::max(mx, out[i]); }
        if (top_db >= 0.f)
            for (int64_t i = 0; i < n; ++i) out[i] = std::max(out[i], mx - top_db);
    });
}


int32_t b2a_weights_sanitize_mimi(b2a_weights* w) {
    return guarded([&] {
        B2A_CHECK(w, B2A_ERR_INVALID_INPUT, "b2a_weights_sanitize_mimi: null handle");
        w->sanitize_mimi();
    });
}

// Mimi.fromPretrained (Mimi.swift:236-335) on a local checkpoint file: mimi_202407(num_codebooks) -> load -> sanitize -> create
int32_t b2a_mimi_create_from_file(const char* path, int32_t num_codebooks, int32_t device, int32_t max_batch, int32_t max_cache_frames,
                                  b2a_mimi** out) {
    return guarded([&] {
        B2A_CHECK(path && out, B2A_ERR_INVALID_INPUT, "b2a_mimi_create_from_file: null argument");
        *out = nullptr;
        b2a_mimi_config cfg{};
        int32_t st = b2a_mimi_config_default(num_codebooks, max_batch, max_cache_frames, &cfg);
        if (st != B2A_OK) throw Error(st, b2a_last_error());
        std::unique_ptr<b2a_weights> w(new b2a_weights());
        w->load_file(path);
        w->sanitize_mimi();
        const std::vector<b2a_tensor> tab = w->table();
        st = b2a_mimi_create(device, &cfg, tab.data(), (int32_t)tab.size(), out);
        if (st != B2A_OK) throw Error(st, b2a_last_error());
    });
}

}  // extern "C"
