// model_file.cc — the reference's config::Model text protos (examples/*/net.pbtxt, read by ReadPbtxt, src/util.cc:87):
// ReadModelText parses one as protobuf's TextFormat does for these messages and maps it onto a ModelConfig with the
// reference's semantics, for a model file (ReadModelFile) and for the text of a built-in model (models.cc) alike;
// ModelText prints any ModelConfig as one.  Protobuf is not a dependency: the schema below is
// proto/convnet_config.proto's field names, types and presence rules.
#include <algorithm>
#include <cctype>
#include <cerrno>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <map>
#include <memory>
#include <set>
#include <sstream>
#include <stdexcept>
#include <tuple>

#include "convnet.h"

namespace cnbhost {

namespace {

// ---------------------------------------------------------------- schema (proto/convnet_config.proto)
// per message: "name:type" entries; type i int32, f float, b bool, s string, else an enum or message name.
// A '!' after the name marks a required field, a '*' a repeated one.
const std::map<std::string, std::string> kMessages = {
    {"Model", "name!:s layer*:Layer edge*:Edge seed!:i max_iter:i display_after:i save_after:i image_size:i patch_size:i "
              "print_after:i localizer:b checkpoint_dir:s print_weights:b timestamp*:s display:b validate_after:i "
              "reduce_lr_factor:f reduce_lr_threshold:f reduce_lr_num_steps:i reduce_lr_max:i smaller_is_better:b "
              "polyak_after:i polyak_queue_size:i subnet*:Subnet train_dataset:DatasetConfig valid_dataset:DatasetConfig "
              "default_weight_optimizer:Optimizer default_bias_optimizer:Optimizer reduce_lr_layer_name:s"},
    {"Layer", "name!:s num_channels:i size:i dropprob:f is_input:b activation:Activation image_size_y:i image_size_x:i "
              "display:b is_output:b gaussian_dropout:b max_act_gaussian_dropout:f gpu_id:i hinge_margin:f "
              "layer_slice*:LayerSlice loss_function:LossFunction performance_metric:LossFunction loss_function_weight:f "
              "tied_data:s image_size_t:i batch_normalize:b bn_f:f bn_epsilon:f gamma_optimizer:Optimizer "
              "beta_optimizer:Optimizer"},
    {"LayerSlice", "name!:s num_channels:i"},
    {"Optimizer", "optimizer_type:OptimizerType epsilon:f epsilon_decay_timescale:i initial_momentum:f final_momentum:f "
                  "momentum_transition_timescale:i l2_decay:f weight_norm_limit:f weight_norm_constraint:f "
                  "epsilon_decay:Decay minimum_epsilon:f decay_factor:f gradient_clip:f lbfgs_memory:i "
                  "start_optimization_after:i adagrad_delta:f rms_prop_factor:f nesterov_momentum:b shared_prior:b "
                  "shared_prior_cost:f shared_prior_file:s"},
    {"Edge", "source!:s dest!:s edge_type:EdgeType kernel_size:i stride:i padding:i initialization:Initialization "
             "init_wt:f init_bias:f weight_optimizer:Optimizer bias_optimizer:Optimizer shared_bias:b block_backprop:b "
             "tied_to:s has_no_bias:b scale_gradients:f partial_sum:i sample_factor:i response_norm_in_blocks:b "
             "add_scale:f pow_scale:f frac_of_filters_response_norm:f gpu_id:i pretrained_model:s pretrained_edge_name:s "
             "display:b source_slice:s dest_slice:s grad_check:b grad_check_num_params:i grad_check_epsilon*:f "
             "kernel_size_y:i kernel_size_x:i kernel_size_t:i stride_y:i stride_x:i stride_t:i padding_y:i padding_x:i "
             "padding_t:i"},
    {"Subnet", "name!:s model_file!:s parameters_file:s merge_layer*:MergeLayer block_backprop:b "
               "start_optimization_after:i gpu_id_offset:i num_channels_multiplier:i remove_layer*:s"},
    {"MergeLayer", "subnet_layer!:s net_layer!:s"},
    {"DataStreamConfig", "file_pattern!:s layer_name!:s dataset_name:s data_type:DataType raw_image_size:i image_size:i "
                         "can_translate:b can_flip:b pixelwise_normalize:b pca_noise_stddev:f normalize:b gpu_id:i "
                         "stride:i mean_file:s num_colors:i parallel_disk_access:b jitter_raw_image:b "
                         "random_rotate_max_angle:f min_scale:f noise_layer_name:s avg10_full_image:b bbox_file:s "
                         "context_factor:f center_on_bbox:b warp_bbox:b gpu_image_size_y:i gpu_image_size_x:i "
                         "raw_image_size_y:i raw_image_size_x:i image_size_y:i image_size_x:i is_sequence:b "
                         "seq_length:i boundary_file:s pick_first:b normalize_local:b"},
    {"DatasetConfig", "data_config*:DataStreamConfig batch_size:i chunk_size:i max_reuse_count:i pipeline_loads:b "
                      "randomize_cpu:b randomize_gpu:b random_access_chunk_size:i max_dataset_size:i multiplicity:i"},
};
// enum values in number order (every enum of the file numbers its values 0, 1, 2, ...)
const std::map<std::string, std::string> kEnums = {
    {"Activation", "LINEAR LOGISTIC RECTIFIED_LINEAR SOFTMAX SOFTMAX_DIST"},
    {"LossFunction", "SQUARED_ERROR LINEAR_ERROR CROSS_ENTROPY_MULTINOMIAL CROSS_ENTROPY_BINARY "
                     "CROSS_ENTROPY_MULTINOMIAL_DISTRIBUTED CLASSIFICATION_MULTINOMIAL CLASSIFICATION_BINARY HINGE_LINEAR "
                     "HINGE_QUADRATIC"},
    {"OptimizerType", "STOCHASTIC_GRADIENT_DESCENT LBFGS ADAGRAD_SGD RMSPROP_SGD"},
    {"Decay", "NONE INVERSE_T EXPONENTIAL LINEAR EXPONENTIAL_STEP"},
    {"EdgeType", "FC CONVOLUTIONAL LOCAL MAXPOOL RESPONSE_NORM UPSAMPLE DOWNSAMPLE RGBTOYUV AVERAGE_POOL CONV_ONETOONE"},
    {"Initialization", "DENSE_GAUSSIAN SPARSE_GAUSSIAN CONSTANT DENSE_GAUSSIAN_SQRT_FAN_IN PRETRAINED DENSE_UNIFORM "
                       "DENSE_UNIFORM_SQRT_FAN_IN"},
    {"DataType", "DUMMY HDF5 IMAGE_RAW SLIDING_WINDOW TXT BOUNDING_BOX CROPS VIDEO_RAW"},
};

std::vector<std::string> Words(const std::string& s) {
  std::istringstream in(s);
  std::vector<std::string> w;
  for (std::string x; in >> x;) w.push_back(x);
  return w;
}
const std::vector<std::string>& EnumValues(const std::string& e) {
  static const std::map<std::string, std::vector<std::string>> all = [] {
    std::map<std::string, std::vector<std::string>> m;
    for (const auto& [name, values] : kEnums) m[name] = Words(values);
    return m;
  }();
  return all.at(e);
}

enum Kind { INT, FLOAT, BOOL, STRING, ENUM, MESSAGE };
struct FieldSpec { Kind kind; std::string type; bool required, repeated; };
const std::map<std::string, FieldSpec>& Schema(const std::string& message) {
  static const std::map<std::string, std::map<std::string, FieldSpec>> all = [] {
    const std::map<std::string, Kind> scalar = {{"i", INT}, {"f", FLOAT}, {"b", BOOL}, {"s", STRING}};
    std::map<std::string, std::map<std::string, FieldSpec>> m;
    for (const auto& [type, fields] : kMessages)
      for (const std::string& w : Words(fields)) {
        const size_t colon = w.find(':');
        std::string name = w.substr(0, colon);
        FieldSpec f{MESSAGE, w.substr(colon + 1), false, false};
        if (name.back() == '!') { f.required = true; name.pop_back(); }
        if (name.back() == '*') { f.repeated = true; name.pop_back(); }
        if (scalar.count(f.type)) f.kind = scalar.at(f.type);
        else if (kEnums.count(f.type)) f.kind = ENUM;
        m[type][name] = f;
      }
    return m;
  }();
  return all.at(message);
}

// ---------------------------------------------------------------- parsed message: fields in file order, with lines
struct Msg;
struct Entry {
  std::string name;
  std::string file;          // the file the line is in (a subnet's fields come from the subnet's model file)
  int line = 0;
  long long i = 0;           // INT, BOOL, ENUM (the value's number)
  float f = 0.f;             // FLOAT
  std::string s;             // STRING, ENUM (the value's name)
  std::shared_ptr<Msg> msg;  // MESSAGE
};
struct Msg {
  std::string type;
  int line = 0;              // of the field that opened it (1 for the file)
  std::vector<Entry> fields;
  const Entry* Get(const std::string& name) const {        // a non-repeated field, nullptr if absent
    for (const Entry& e : fields) if (e.name == name) return &e;
    return nullptr;
  }
  bool Has(const std::string& name) const { return Get(name) != nullptr; }
  long long Int(const std::string& name, long long def) const { const Entry* e = Get(name); return e ? e->i : def; }
  float Float(const std::string& name, float def) const { const Entry* e = Get(name); return e ? e->f : def; }
  bool Bool(const std::string& name, bool def) const { const Entry* e = Get(name); return e ? e->i != 0 : def; }
  std::string Enum(const std::string& name, const std::string& def) const { const Entry* e = Get(name); return e ? e->s : def; }
  std::vector<const Entry*> All(const std::string& name) const {
    std::vector<const Entry*> out;
    for (const Entry& e : fields) if (e.name == name) out.push_back(&e);
    return out;
  }
};

// ---------------------------------------------------------------- tokenizer and parser (TextFormat)
class Parser {
 public:
  Parser(const std::string& path, const std::string& text) : path_(path), t_(text) {}

  std::shared_ptr<Msg> ParseFile() {
    auto m = std::make_shared<Msg>();
    m->type = "Model"; m->line = 1;
    ParseBody(*m, '\0');
    return m;
  }

 private:
  enum Tok { END, IDENT, NUMBER, STR, SYMBOL };
  const std::string path_, t_;
  size_t p_ = 0;
  int line_ = 1;
  Tok tok_ = END;
  std::string text_;         // IDENT / NUMBER: as written; STR: the decoded bytes; SYMBOL: the character
  int tok_line_ = 1;
  bool peeked_ = false;

  [[noreturn]] void Fail(int line, const std::string& what) const {
    throw std::invalid_argument(path_ + ":" + std::to_string(line) + ": " + what);
  }
  void SkipSpace() {
    while (p_ < t_.size()) {
      const char c = t_[p_];
      if (c == '\n') { line_++; p_++; }
      else if (c == ' ' || c == '\t' || c == '\r' || c == '\v' || c == '\f') p_++;
      else if (c == '#') { while (p_ < t_.size() && t_[p_] != '\n') p_++; }
      else break;
    }
  }
  static bool IdentStart(char c) { return (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || c == '_'; }
  static bool Digit(char c) { return c >= '0' && c <= '9'; }
  // the next token, without consuming it
  Tok Peek() {
    if (peeked_) return tok_;
    peeked_ = true;
    SkipSpace();
    tok_line_ = line_;
    text_.clear();
    if (p_ >= t_.size()) return tok_ = END;
    const char c = t_[p_];
    if (IdentStart(c)) {
      while (p_ < t_.size() && (IdentStart(t_[p_]) || Digit(t_[p_]))) text_ += t_[p_++];
      return tok_ = IDENT;
    }
    if (Digit(c) || (c == '.' && p_ + 1 < t_.size() && Digit(t_[p_ + 1]))) {
      while (p_ < t_.size() && (IdentStart(t_[p_]) || Digit(t_[p_]) || t_[p_] == '.' ||
                                ((t_[p_] == '+' || t_[p_] == '-') && (t_[p_ - 1] == 'e' || t_[p_ - 1] == 'E') &&
                                 !(text_.size() > 1 && (text_[1] == 'x' || text_[1] == 'X')))))
        text_ += t_[p_++];
      return tok_ = NUMBER;
    }
    if (c == '"' || c == '\'') {
      p_++;
      while (true) {                                       // one or more adjacent literals, concatenated
        ReadString(t_[p_ - 1]);
        const size_t save_p = p_; const int save_line = line_;
        SkipSpace();
        if (p_ < t_.size() && (t_[p_] == '"' || t_[p_] == '\'')) { p_++; continue; }
        p_ = save_p; line_ = save_line;
        break;
      }
      return tok_ = STR;
    }
    text_ = std::string(1, c);
    p_++;
    return tok_ = SYMBOL;
  }
  // the body of a string literal opened by `quote` (already consumed), escapes decoded, appended to text_
  void ReadString(char quote) {
    while (true) {
      if (p_ >= t_.size() || t_[p_] == '\n') Fail(tok_line_, "string literal not closed");
      const char c = t_[p_++];
      if (c == quote) return;
      if (c != '\\') { text_ += c; continue; }
      if (p_ >= t_.size()) Fail(line_, "string literal not closed");
      const char e = t_[p_++];
      static const std::string from = "ntrabfv\\'\"?", to = "\n\t\r\a\b\f\v\\'\"?";
      const size_t k = from.find(e);
      if (k != std::string::npos) { text_ += to[k]; continue; }
      if (e >= '0' && e <= '7') {                          // up to three octal digits
        int v = e - '0';
        for (int n = 1; n < 3 && p_ < t_.size() && t_[p_] >= '0' && t_[p_] <= '7'; n++) v = 8 * v + (t_[p_++] - '0');
        text_ += (char)v;
        continue;
      }
      if (e == 'x' || e == 'X') {                          // up to two hex digits
        int v = 0, n = 0;
        for (; n < 2 && p_ < t_.size() && isxdigit((unsigned char)t_[p_]); n++)
          v = 16 * v + (Digit(t_[p_]) ? t_[p_] - '0' : (tolower(t_[p_]) - 'a' + 10)), p_++;
        if (!n) Fail(line_, "\\x without hex digits in a string literal");
        text_ += (char)v;
        continue;
      }
      Fail(line_, std::string("invalid escape \\") + e + " in a string literal");
    }
  }
  Tok Next() { Tok k = Peek(); peeked_ = false; return k; }
  bool TrySymbol(char c) {
    if (Peek() == SYMBOL && text_[0] == c) { Next(); return true; }
    return false;
  }
  std::string Describe() {
    switch (Peek()) {
      case END: return "end of file";
      case STR: return "a string";
      default: return "'" + text_ + "'";
    }
  }

  // fields until `close` ('}' or '>'; '\0': end of file)
  void ParseBody(Msg& m, char close) {
    const std::map<std::string, FieldSpec>& schema = Schema(m.type);
    std::set<std::string> seen;
    while (true) {
      if (close == '\0' ? Peek() == END : TrySymbol(close)) break;
      if (Peek() == END) Fail(line_, "'" + m.type + "' block opened on line " + std::to_string(m.line) + " is not closed");
      if (Peek() != IDENT) Fail(tok_line_, "expected a field name of '" + m.type + "', found " + Describe());
      const std::string name = text_;
      const int line = tok_line_;
      Next();
      auto it = schema.find(name);
      if (it == schema.end()) Fail(line, "unknown field '" + name + "' in '" + m.type + "'");
      const FieldSpec& f = it->second;
      if (!f.repeated && !seen.insert(name).second) Fail(line, "field '" + name + "' is given twice (it is not repeated)");
      if (f.kind == MESSAGE) {
        TrySymbol(':');
        if (TrySymbol('[')) {
          if (!f.repeated) Fail(line, "field '" + name + "': a list for a field that is not repeated");
          if (!TrySymbol(']')) {
            do { ParseMessageValue(m, name, f, line); } while (TrySymbol(','));
            if (!TrySymbol(']')) Fail(tok_line_, "field '" + name + "': expected ',' or ']' in the list, found " + Describe());
          }
        } else {
          ParseMessageValue(m, name, f, line);
        }
      } else {
        if (!TrySymbol(':')) Fail(tok_line_, "field '" + name + "': expected ':', found " + Describe());
        if (TrySymbol('[')) {
          if (!f.repeated) Fail(line, "field '" + name + "': a list for a field that is not repeated");
          if (!TrySymbol(']')) {
            do { m.fields.push_back(ParseScalar(name, f)); } while (TrySymbol(','));
            if (!TrySymbol(']')) Fail(tok_line_, "field '" + name + "': expected ',' or ']' in the list, found " + Describe());
          }
        } else {
          m.fields.push_back(ParseScalar(name, f));
        }
      }
      if (!TrySymbol(',')) TrySymbol(';');
    }
    for (const auto& [name, f] : schema)
      if (f.required && !m.Has(name)) Fail(m.line, "'" + m.type + "' block without its required field '" + name + "'");
  }
  void ParseMessageValue(Msg& m, const std::string& name, const FieldSpec& f, int line) {
    char close;
    if (TrySymbol('{')) close = '}';
    else if (TrySymbol('<')) close = '>';
    else Fail(tok_line_, "field '" + name + "': expected '{', found " + Describe());
    Entry e;
    e.name = name; e.file = path_; e.line = line;
    e.msg = std::make_shared<Msg>();
    e.msg->type = f.type; e.msg->line = line;
    ParseBody(*e.msg, close);
    m.fields.push_back(e);
  }
  Entry ParseScalar(const std::string& name, const FieldSpec& f) {
    Entry e;
    e.name = name;
    e.file = path_;
    e.line = tok_line_;
    auto bad = [&](const std::string& want) { Fail(e.line, "field '" + name + "': expected " + want + ", found " + Describe()); };
    if (f.kind == STRING) {
      if (Peek() != STR) bad("a string");
      e.s = text_;
      Next();
      return e;
    }
    const bool minus = TrySymbol('-');
    if (f.kind == FLOAT) {
      double v;
      if (Peek() == IDENT &&
          (text_ == "inf" || text_ == "Inf" || text_ == "infinity" || text_ == "Infinity" || text_ == "nan" || text_ == "NaN")) {
        v = text_[0] == 'n' || text_[0] == 'N' ? NAN : INFINITY;
      } else {
        if (Peek() != NUMBER) bad("a number");
        std::string s = text_;
        if (s.size() > 1 && (s.back() == 'f' || s.back() == 'F') && s.find_first_of("xX") == std::string::npos) s.pop_back();
        long long iv;
        if (ParseInteger(s, &iv)) v = (double)iv;
        else if (!ParseDecimal(s, &v)) bad("a number");
      }
      Next();
      e.f = (float)(minus ? -v : v);                       // as protobuf: parsed as a double, then rounded to float
      return e;
    }
    if (f.kind == INT) {
      long long v;
      if (Peek() != NUMBER || !ParseInteger(text_, &v)) bad("an integer");
      if (minus) v = -v;
      if (v < -2147483648LL || v > 2147483647LL) Fail(e.line, "field '" + name + "': " + text_ + " is out of the int32 range");
      Next();
      e.i = v;
      return e;
    }
    if (f.kind == BOOL) {
      if (minus) bad("true or false");
      if (Peek() == IDENT && (text_ == "true" || text_ == "True" || text_ == "t")) e.i = 1;
      else if (Peek() == IDENT && (text_ == "false" || text_ == "False" || text_ == "f")) e.i = 0;
      else if (Peek() == NUMBER && (text_ == "0" || text_ == "1")) e.i = text_ == "1";
      else bad("true or false");
      Next();
      return e;
    }
    // ENUM: a value name, or its number
    const std::vector<std::string>& values = EnumValues(f.type);
    long long v = -1;
    if (!minus && Peek() == IDENT) {
      for (size_t k = 0; k < values.size(); k++) if (values[k] == text_) v = (long long)k;
      if (v < 0) Fail(e.line, "field '" + name + "': '" + text_ + "' is not a value of enum " + f.type);
    } else if (Peek() == NUMBER && ParseInteger(text_, &v)) {
      if (minus) v = -v;
      if (v < 0 || v >= (long long)values.size())
        Fail(e.line, "field '" + name + "': " + std::to_string(v) + " is not a value of enum " + f.type);
    } else {
      bad("a value of enum " + f.type);
    }
    Next();
    e.i = v;
    e.s = values[v];
    return e;
  }
  // decimal, 0x hex or 0-prefixed octal, as protobuf's tokenizer reads an integer
  static bool ParseInteger(const std::string& s, long long* out) {
    if (s.empty() || !Digit(s[0])) return false;
    const int base = s.size() > 1 && s[0] == '0' ? ((s[1] == 'x' || s[1] == 'X') ? 16 : 8) : 10;
    const char* b = s.c_str() + (base == 16 ? 2 : 0);
    if (!*b) return false;
    char* end;
    errno = 0;
    const unsigned long long v = strtoull(b, &end, base);
    if (*end || errno == ERANGE || v > (unsigned long long)INT64_MAX) return false;
    if (out) *out = (long long)v;
    return true;
  }
  static bool ParseDecimal(const std::string& s, double* out) {
    if (s.empty() || s.find_first_of("xX") != std::string::npos) return false;
    char* end;
    *out = strtod(s.c_str(), &end);
    return *end == '\0';
  }
};

// ---------------------------------------------------------------- names shared by the reader and the writer
// host enum -> proto value name
const char* const kActivationNames[] = {"LINEAR", "RECTIFIED_LINEAR", "SOFTMAX", "LOGISTIC", "SOFTMAX_DIST"};
template <size_t N>
int HostValue(const char* const (&names)[N], const std::string& name) {
  for (size_t k = 0; k < N; k++) if (name == names[k]) return (int)k;
  return -1;
}

// the Optimizer fields the host keeps, in proto order; `e`: the enum of an int field
struct OptField { const char* name; float OptimizerConfig::*f; int OptimizerConfig::*i; const char* e; };
const OptField kOptFields[] = {
    {"optimizer_type", nullptr, &OptimizerConfig::optimizer_type, "OptimizerType"},
    {"epsilon", &OptimizerConfig::epsilon, nullptr, nullptr},
    {"epsilon_decay_timescale", nullptr, &OptimizerConfig::epsilon_decay_timescale, nullptr},
    {"initial_momentum", &OptimizerConfig::initial_momentum, nullptr, nullptr},
    {"final_momentum", &OptimizerConfig::final_momentum, nullptr, nullptr},
    {"momentum_transition_timescale", nullptr, &OptimizerConfig::momentum_transition_timescale, nullptr},
    {"l2_decay", &OptimizerConfig::l2_decay, nullptr, nullptr},
    {"weight_norm_limit", &OptimizerConfig::weight_norm_limit, nullptr, nullptr},
    {"weight_norm_constraint", &OptimizerConfig::weight_norm_constraint, nullptr, nullptr},
    {"epsilon_decay", nullptr, &OptimizerConfig::epsilon_decay, "Decay"},
    {"minimum_epsilon", &OptimizerConfig::minimum_epsilon, nullptr, nullptr},
    {"decay_factor", &OptimizerConfig::decay_factor, nullptr, nullptr},
    {"gradient_clip", &OptimizerConfig::gradient_clip, nullptr, nullptr},
    {"start_optimization_after", nullptr, &OptimizerConfig::start_optimization_after, nullptr},
    {"adagrad_delta", &OptimizerConfig::adagrad_delta, nullptr, nullptr},
    {"rms_prop_factor", &OptimizerConfig::rms_prop_factor, nullptr, nullptr},
};

bool HasParameters(EdgeType t) { return t == FC || t == CONVOLUTIONAL || t == LOCAL || t == CONV_ONETOONE; }
bool HasConvGeometry(EdgeType t) { return t == CONVOLUTIONAL || t == LOCAL || t == MAXPOOL || t == AVGPOOL; }
bool IsSampling(EdgeType t) { return t == UPSAMPLE || t == DOWNSAMPLE; }

// ---------------------------------------------------------------- Msg -> ModelConfig
class Mapper {
 public:
  Mapper(const std::string& path, bool check_pretrained) : path_(path), check_pretrained_(check_pretrained) {}

  ModelConfig Map(Msg& model) {
    std::vector<std::string> open = {path_};
    ExpandSubnets(model, open);
    ModelConfig m;
    m.name = model.Get("name")->s;
    m.seed = (unsigned)model.Int("seed", 0);
    // Polyak averaging: a queue without an insertion period, or a period without a queue, averages nothing
    m.polyak_after = (int)model.Int("polyak_after", 0);
    m.polyak_queue_size = (int)model.Int("polyak_queue_size", 0);
    for (int k = 0; k < 2; k++) {
      const char *f = k ? "polyak_queue_size" : "polyak_after", *other = k ? "polyak_after" : "polyak_queue_size";
      if (model.Int(f, 0) > 0 && model.Int(other, 0) <= 0)
        Fail(*model.Get(f), "", std::string("field '") + f + "': Polyak averaging needs both polyak_after and "
             "polyak_queue_size > 0, and " + other + " is not");
    }
    m.validate_after = (int)model.Int("validate_after", -1);
    m.save_after = (int)model.Int("save_after", -1);
    if (PolyakOn(m))                                       // the insertion rule (PolyakDue) divides by both
      for (const char* f : {"validate_after", "save_after"})
        if (model.Int(f, -1) == 0) Fail(*model.Get(f), "", std::string("field '") + f + "': 0 with Polyak averaging on "
                                        "(its insertion rule takes the iteration modulo " + f + ")");
    // the rest of the training schedule (ConvNet::Train checks it when a run starts)
    m.max_iter = (int)model.Int("max_iter", -1);
    m.print_after = (int)model.Int("print_after", -1);
    m.reduce_lr_factor = model.Float("reduce_lr_factor", 1.f);
    m.reduce_lr_threshold = model.Float("reduce_lr_threshold", 0.f);
    m.reduce_lr_num_steps = (int)model.Int("reduce_lr_num_steps", 0);
    m.reduce_lr_max = (int)model.Int("reduce_lr_max", 0);
    m.smaller_is_better = model.Bool("smaller_is_better", false);
    if (const Entry* e = model.Get("reduce_lr_layer_name")) m.reduce_lr_layer_name = e->s;
    if (const Entry* e = model.Get("checkpoint_dir")) m.checkpoint_dir = e->s;
    def_w_ =model.Get("default_weight_optimizer");
    def_b_ = model.Get("default_bias_optimizer");
    for (const Entry* d : {def_w_, def_b_}) if (d) CheckOptimizer(*d, "");

    // the graph (ConvNet::BuildNet, src/convnet.cc:150-220): no incoming edge = input, no outgoing edge = output
    const std::vector<const Entry*> layers = model.All("layer"), edges = model.All("edge");
    if (layers.empty()) Fail(1, "the model has no layer");
    std::map<std::string, size_t> index;
    for (size_t k = 0; k < layers.size(); k++) {
      const std::string& name = layers[k]->msg->Get("name")->s;
      if (!index.emplace(name, k).second) Fail(*layers[k], "layer '" + name + "'", "a second layer of that name");
    }
    std::vector<int> in(layers.size(), -1), out(layers.size(), -1);
    for (size_t k = 0; k < edges.size(); k++) {
      const Msg& e = *edges[k]->msg;
      const std::string where = EdgeName(e);
      size_t end[2];
      for (int d = 0; d < 2; d++) {
        const char* field = d ? "dest" : "source";
        auto it = index.find(e.Get(field)->s);
        if (it == index.end()) Fail(*e.Get(field), where, std::string("field '") + field + "': no layer of that name");
        end[d] = it->second;
      }
      if (out[end[0]] >= 0)
        Fail(*edges[k], where, "layer '" + e.Get("source")->s + "' has a second outgoing edge: the net is not a single chain");
      if (in[end[1]] >= 0)
        Fail(*edges[k], where, "layer '" + e.Get("dest")->s + "' has a second incoming edge: the net is not a single chain");
      out[end[0]] = (int)k; in[end[1]] = (int)k;
    }
    std::vector<size_t> chain;
    for (size_t k = 0; k < layers.size(); k++) if (in[k] < 0) chain.push_back(k);
    if (chain.size() != 1) {
      std::string names;
      for (size_t k : chain) names += (names.empty() ? "'" : ", '") + layers[k]->msg->Get("name")->s + "'";
      Fail(chain.empty() ? *layers[0] : *layers[chain[1]], "",
           chain.empty() ? "every layer has an incoming edge: the net is not a single chain"
                         : "more than one layer without an incoming edge (" + names + "): the net is not a single chain");
    }
    // every layer has at most one incoming edge, so the walk from the input cannot enter a cycle: it ends, and the
    // layers it misses form cycles of their own
    while (out[chain.back()] >= 0) chain.push_back(index.at(edges[out[chain.back()]]->msg->Get("dest")->s));
    if (chain.size() != layers.size()) {
      const std::set<size_t> on(chain.begin(), chain.end());
      for (size_t k = 0; k < layers.size(); k++)
        if (!on.count(k))
          Fail(*layers[k], "layer '" + layers[k]->msg->Get("name")->s + "'",
               "not on the chain that starts at the input layer: the net is not a single chain");
    }
    if (chain.size() < 2) Fail(*layers[chain[0]], "", "the model has no edge");

    for (size_t k = 0; k < chain.size(); k++)
      m.layer.push_back(MapLayer(*layers[chain[k]], k == 0, k + 1 == chain.size()));
    for (size_t k = 0; k + 1 < chain.size(); k++) m.edge.push_back(MapEdge(*edges[out[chain[k]]], m.layer[k]));
    // the data sets' batch order, and the crop of the data stream that feeds the input layer (DataHandler); not written
    // back by model_text
    for (auto [field, spec] : {std::pair{"train_dataset", &m.train_dataset}, std::pair{"valid_dataset", &m.valid_dataset}}) {
      const Entry* d = model.Get(field);
      if (!d) continue;
      const Msg& ds = *d->msg;
      DatasetOrder& o = spec->order;
      spec->present = true;
      o.batch_size = (int)ds.Int("batch_size", 1);
      o.chunk_size = (int)ds.Int("chunk_size", 0);
      o.max_reuse_count = (int)ds.Int("max_reuse_count", 0);
      o.pipeline_loads = ds.Bool("pipeline_loads", false);
      o.randomize_cpu = ds.Bool("randomize_cpu", false);
      o.randomize_gpu = ds.Bool("randomize_gpu", false);
      o.random_access_chunk_size = (int)ds.Int("random_access_chunk_size", 1);
      o.multiplicity = (int)ds.Int("multiplicity", 1);
      for (const Entry* s : ds.All("data_config")) {
        const Msg& dc = *s->msg;
        if (dc.Get("layer_name")->s != m.layer.front().name) continue;
        spec->translate = dc.Bool("can_translate", false);
        spec->flip = dc.Bool("can_flip", false);
        spec->gpu_image_size_y = (int)dc.Int("gpu_image_size_y", 0);
        spec->gpu_image_size_x = (int)dc.Int("gpu_image_size_x", 0);
        break;
      }
    }
    // what needs the whole chain: ConvNet's checks, at the line of the first field the refusal names that the layer or edge
    // block sets (else of the block), then the checkpoints of the PRETRAINED edges
    std::unique_ptr<ConvNet> net;
    try {
      net = std::make_unique<ConvNet>(m, 1);               // host only: no device memory
    } catch (const ModelRefused& r) {
      const Entry& block = r.edge ? *edges[out[chain[r.index]]] : *layers[chain[r.index]];
      const Entry* at = &block;
      for (const std::string& f : r.fields)
        if (const Entry* e = block.msg->Get(f)) { at = e; break; }
      Fail(*at, "", r.what());
    }
    for (size_t k = 0; check_pretrained_ && k < m.edge.size(); k++) {
      const Edge& e = *net->Edges()[k];
      if (m.edge[k].initialization == PRETRAINED && !e.HasNoParameters() && m.edge[k].tied_to.empty())
        CheckPretrained(*edges[out[chain[k]]]->msg, dynamic_cast<const EdgeWithWeight&>(e), m.edge[k]);
    }
    return m;
  }

 private:
  const std::string path_;
  const bool check_pretrained_;
  const Entry *def_w_ = nullptr, *def_b_ = nullptr;

  // a PRETRAINED edge (shapes known): its checkpoint has the weight and bias records, with their optimizers' history and
  // step, at this edge's sizes (EdgeWithWeight::LoadParameters, edge_with_weight.cc:41-58)
  void CheckPretrained(const Msg& e, const EdgeWithWeight& w, const EdgeConfig& c) const {
    const std::string where = EdgeName(e);
    const Entry& file = *e.Get("pretrained_model");
    std::unique_ptr<CheckpointFile> f;
    try {
      f.reset(new CheckpointFile(c.pretrained_model));
    } catch (const std::invalid_argument& x) {
      Fail(file, where, std::string("field 'pretrained_model': ") + x.what());
    }
    const Entry& field = e.Has("pretrained_edge_name") ? *e.Get("pretrained_edge_name") : file;
    const std::string from = c.pretrained_edge_name.empty() ? c.name : c.pretrained_edge_name;
    for (int which = 0; which < 2; which++) {
      const long long n = which ? w.BiasCount() : w.WeightCount();
      if (n == 0) continue;
      const std::string prefix = from + (which ? ":bias" : ":weight");
      for (const auto& [name, type, count] : {std::make_tuple(prefix, (int)CheckpointFile::FLOAT32, n),
                                              std::make_tuple(prefix + "_gradient_history", (int)CheckpointFile::FLOAT32, n),
                                              std::make_tuple(prefix + "_step", (int)CheckpointFile::INT64, 1LL)}) {
        const std::string why = f->Check(name, type, count);
        if (!why.empty()) Fail(field, where, "field '" + field.name + "': " + why);
      }
    }
  }

  [[noreturn]] void Fail(int line, const std::string& what) const {
    throw std::invalid_argument(path_ + ":" + std::to_string(line) + ": " + what);
  }
  // "<where>: field '<name>': <what>" at the field's line
  [[noreturn]] void Fail(const Entry& at, const std::string& where, const std::string& what) const {
    throw std::invalid_argument(at.file + ":" + std::to_string(at.line) + ": " + (where.empty() ? "" : where + ": ") + what);
  }
  void RefuseMessage(const Msg& m, const char* field, const std::string& why, const std::string& where = "") const {
    if (const Entry* e = m.Get(field)) Fail(*e, where, std::string("field '") + field + "': " + why);
  }
  static std::string EdgeName(const Msg& e) { return "edge '" + e.Get("source")->s + ":" + e.Get("dest")->s + "'"; }

  // ---- subnets (ConvNet::AddSubnet, src/convnet.cc:94-148): the layers and edges of each subnet join `model` before its
  // graph is mapped, and the subnet blocks go (convnet.cc:39).  `open`: the model files being expanded, outermost first
  void ExpandSubnets(Msg& model, std::vector<std::string>& open) const {
    std::vector<Entry> subnets;
    for (const Entry& e : model.fields) if (e.name == "subnet") subnets.push_back(e);
    model.fields.erase(std::remove_if(model.fields.begin(), model.fields.end(), [](const Entry& e) { return e.name == "subnet"; }),
                       model.fields.end());
    for (const Entry& s : subnets) AddSubnet(model, s, open);
  }
  // field v.name of `m` set to `v`
  static void Set(Msg& m, const Entry& v) {
    for (Entry& e : m.fields) if (e.name == v.name) { e = v; return; }
    m.fields.push_back(v);
  }
  // a field that a subnet block sets, at the line of `at`
  static Entry Value(const Entry& at, const std::string& name) {
    Entry e;
    e.name = name; e.file = at.file; e.line = at.line;
    return e;
  }
  void AddSubnet(Msg& model, const Entry& at, std::vector<std::string>& open) const {
    const Msg& s = *at.msg;
    const std::string name = s.Get("name")->s, where = "subnet '" + name + "'";
    const Entry& file = *s.Get("model_file");
    if (s.Int("gpu_id_offset", 0) != 0)
      Fail(*s.Get("gpu_id_offset"), where, "field 'gpu_id_offset': one GPU per model (data parallelism replicates it)");
    const long long mult = s.Int("num_channels_multiplier", 1);
    if (mult <= 0) Fail(*s.Get("num_channels_multiplier"), where, "field 'num_channels_multiplier' must be positive");
    if (std::find(open.begin(), open.end(), file.s) != open.end())
      Fail(file, where, "field 'model_file': '" + file.s + "' contains itself as a subnet");
    std::ifstream in(file.s, std::ios::binary);
    if (!in) Fail(file, where, "field 'model_file': cannot open model file '" + file.s + "'");
    std::stringstream text;
    text << in.rdbuf();
    const std::shared_ptr<Msg> sub = Parser(file.s, text.str()).ParseFile();
    open.push_back(file.s);
    ExpandSubnets(*sub, open);                             // its own subnets first
    open.pop_back();

    std::set<std::string> sub_layers, net_layers;
    for (const Entry* l : sub->All("layer")) sub_layers.insert(l->msg->Get("name")->s);
    for (const Entry* l : model.All("layer")) net_layers.insert(l->msg->Get("name")->s);
    // the reference ignores a merge_layer or remove_layer that names no layer of the subnet; here it is refused
    std::map<std::string, std::string> merge;
    for (const Entry* ml : s.All("merge_layer")) {
      const Entry &from = *ml->msg->Get("subnet_layer"), &to = *ml->msg->Get("net_layer");
      if (!sub_layers.count(from.s)) Fail(from, where, "field 'subnet_layer': " + file.s + " has no layer '" + from.s + "'");
      if (!net_layers.count(to.s)) Fail(to, where, "field 'net_layer': the net has no layer '" + to.s + "'");
      merge[from.s] = to.s;
    }
    std::set<std::string> removed;
    for (const Entry* r : s.All("remove_layer")) {
      if (!sub_layers.count(r->s)) Fail(*r, where, "field 'remove_layer': " + file.s + " has no layer '" + r->s + "'");
      removed.insert(r->s);
    }
    auto renamed = [&](const std::string& l) { return merge.count(l) ? merge.at(l) : name + "_" + l; };

    for (const Entry* l : sub->All("layer")) {              // a merged layer takes the net's config: the subnet's goes
      const std::string& old = l->msg->Get("name")->s;
      if (merge.count(old) || removed.count(old)) continue;
      Entry layer = *l;
      layer.msg = std::make_shared<Msg>(*l->msg);
      Entry n = *layer.msg->Get("name");
      n.s = renamed(old);
      if (!net_layers.insert(n.s).second) Fail(*l, where, "layer '" + old + "' becomes '" + n.s + "', a layer the net already has");
      Set(*layer.msg, n);
      if (const Entry* c = layer.msg->Get("num_channels")) {
        Entry v = *c;
        v.i *= mult;
        if (v.i > 2147483647LL) Fail(*c, where, "field 'num_channels': " + std::to_string(v.i) + " channels after the multiplier");
        Set(*layer.msg, v);
      }
      model.fields.push_back(layer);
    }

    std::map<std::string, std::string> edge_names;          // subnet edge -> its name in the net (tied_to)
    for (const Entry* e : sub->All("edge")) {
      const std::string &src = e->msg->Get("source")->s, &dst = e->msg->Get("dest")->s;
      if (!removed.count(src) && !removed.count(dst)) edge_names[src + ":" + dst] = renamed(src) + ":" + renamed(dst);
    }
    const Entry* params = s.Get("parameters_file");
    const Entry* block = s.Bool("block_backprop", false) ? s.Get("block_backprop") : nullptr;
    const Entry& soa = s.Has("start_optimization_after") ? *s.Get("start_optimization_after") : at;
    for (const Entry* e : sub->All("edge")) {
      const std::string src = e->msg->Get("source")->s, dst = e->msg->Get("dest")->s;
      if (removed.count(src) || removed.count(dst)) continue;
      Entry edge = *e;
      edge.msg = std::make_shared<Msg>(*e->msg);
      Msg& m = *edge.msg;
      if (params && !params->s.empty()) {                  // PRETRAINED from the checkpoint, by the edge's subnet name
        Entry v = Value(*params, "initialization");
        v.i = PRETRAINED; v.s = "PRETRAINED";
        Set(m, v);
        v = Value(*params, "pretrained_model"); v.s = params->s; Set(m, v);
        v = Value(*params, "pretrained_edge_name"); v.s = src + ":" + dst; Set(m, v);
      }
      for (const char* f : {"source", "dest"}) {
        Entry v = *m.Get(f);
        v.s = renamed(v.s);
        Set(m, v);
      }
      // the reference leaves tied_to as the subnet wrote it, naming an edge the net does not have
      if (const Entry* tie = m.Get("tied_to"); tie && edge_names.count(tie->s)) {
        Entry v = *tie;
        v.s = edge_names.at(tie->s);
        Set(m, v);
      }
      if (block && !m.Bool("block_backprop", false)) {
        Entry v = Value(*block, "block_backprop");
        v.i = 1;
        Set(m, v);
      }
      for (const char* f : {"weight_optimizer", "bias_optimizer"}) {
        Entry o = m.Has(f) ? *m.Get(f) : Value(soa, f);
        o.msg = o.msg ? std::make_shared<Msg>(*o.msg) : std::make_shared<Msg>();
        if (!m.Has(f)) { o.msg->type = "Optimizer"; o.msg->line = soa.line; }
        Entry v = Value(soa, "start_optimization_after");
        v.i = s.Int("start_optimization_after", 0);
        Set(*o.msg, v);
        Set(m, o);
      }
      model.fields.push_back(edge);
    }
  }

  // Optimizer fields outside the SGD / Adagrad / RMSProp paths: refused wherever a block sets them
  void CheckOptimizer(const Entry& block, const std::string& where) const {
    const Msg& o = *block.msg;
    const std::string w = (where.empty() ? "" : where + ": ") + block.name;
    auto refuse = [&](const char* f, const char* why) { Fail(*o.Get(f), w, std::string("field '") + f + "': " + why); };
    if (o.Int("lbfgs_memory", 0) != 0) refuse("lbfgs_memory", "LBFGS is not supported");
    if (o.Bool("nesterov_momentum", false)) refuse("nesterov_momentum", "Nesterov momentum is not supported");
    if (o.Bool("shared_prior", false)) refuse("shared_prior", "shared priors are not supported");
    if (o.Float("shared_prior_cost", 0.f) != 0.f) refuse("shared_prior_cost", "shared priors are not supported");
    if (o.Has("shared_prior_file")) refuse("shared_prior_file", "shared priors are not supported");
  }
  // config::Optimizer d(default); d.MergeFrom(own): every field present in `own` overrides (src/convnet.cc:45-52)
  OptimizerConfig Merge(const Entry* def, const Entry* own, const std::string& where) const {
    OptimizerConfig c;
    for (const Entry* block : {def, own}) {
      if (!block) continue;
      for (const OptField& f : kOptFields) {
        const Entry* e = block->msg->Get(f.name);
        if (!e) continue;
        if (f.f) c.*f.f = e->f;
        else c.*f.i = (int)e->i;
      }
    }
    if (const char* err = OptimizerConfigError(c)) {
      if (const Entry* at = own ? own : def) Fail(*at, where, at->name + ": " + err);
      Fail(1, where + ": optimizer: " + err);
    }
    return c;
  }

  LayerConfig MapLayer(const Entry& at, bool input, bool output) const {
    const Msg& l = *at.msg;
    LayerConfig c;
    c.name = l.Get("name")->s;
    const std::string where = "layer '" + c.name + "'";
    RefuseMessage(l, "layer_slice", "layer slices are not supported", where);
    RefuseMessage(l, "tied_data", "tied data is not supported", where);
    if (l.Bool("gaussian_dropout", false)) Fail(*l.Get("gaussian_dropout"), where, "field 'gaussian_dropout': not supported");
    if (l.Int("gpu_id", 0) != 0) Fail(*l.Get("gpu_id"), where, "field 'gpu_id': one GPU per model (data parallelism replicates it)");
    c.num_channels = (int)l.Int("num_channels", 0);
    if (c.num_channels <= 0) Fail(l.Has("num_channels") ? *l.Get("num_channels") : at, where, "field 'num_channels' must be positive");
    c.is_input = input;                                    // is_input / is_output (deprecated) are not read
    c.is_output = output;
    c.activation = (Activation)HostValue(kActivationNames, l.Enum("activation", "LINEAR"));
    c.dropprob = l.Float("dropprob", 0.f);
    c.loss_function = (int)l.Int("loss_function", CROSS_ENTROPY_MULTINOMIAL);
    c.performance_metric = (int)l.Int("performance_metric", CLASSIFICATION_MULTINOMIAL);
    c.loss_function_weight = l.Float("loss_function_weight", 1.f);
    if (input) {
      c.image_size_y = (int)l.Int("image_size_y", 1);
      c.image_size_x = (int)l.Int("image_size_x", 1);
      c.image_size_t = (int)l.Int("image_size_t", 1);
      if (c.image_size_y <= 0 || c.image_size_x <= 0 || c.image_size_t <= 0)
        Fail(at, where, "fields 'image_size_y' / 'image_size_x' / 'image_size_t' must be positive");
    }
    c.batch_normalize = l.Bool("batch_normalize", false);
    c.bn_f = l.Float("bn_f", 0.98f);
    c.bn_epsilon = l.Float("bn_epsilon", 1e-5f);
    if (c.batch_normalize) {
      // gamma merges with the default weight optimizer and beta with the default bias optimizer (DESIGN.md §5)
      for (const char* f : {"gamma_optimizer", "beta_optimizer"}) if (const Entry* e = l.Get(f)) CheckOptimizer(*e, where);
      c.gamma_optimizer = Merge(def_w_, l.Get("gamma_optimizer"), where);
      c.beta_optimizer = Merge(def_b_, l.Get("beta_optimizer"), where);
    }
    return c;
  }

  EdgeConfig MapEdge(const Entry& at, const LayerConfig& source) const {
    const Msg& e = *at.msg;
    const std::string where = EdgeName(e);
    EdgeConfig c;
    c.source = e.Get("source")->s;
    c.dest = e.Get("dest")->s;
    c.name = c.source + ":" + c.dest;
    const std::string type = e.Enum("edge_type", "FC");
    const int t = HostValue(kEdgeTypeNames, type);
    if (t < 0) Fail(*e.Get("edge_type"), where, "field 'edge_type': " + type + " is not supported");
    c.edge_type = (EdgeType)t;
    if (const Entry* tie = e.Get("tied_to")) c.tied_to = tie->s;
    RefuseMessage(e, "source_slice", "layer slices are not supported", where);
    RefuseMessage(e, "dest_slice", "layer slices are not supported", where);
    c.block_backprop = e.Bool("block_backprop", false);
    if (e.Int("gpu_id", 0) != 0) Fail(*e.Get("gpu_id"), where, "field 'gpu_id': one GPU per model (data parallelism replicates it)");

    // geometry: the *_y / *_x fields fall back to kernel_size / stride / padding only when absent (src/edge.cc:87-106)
    c.kernel_size = (int)e.Int("kernel_size", -1);
    c.stride = (int)e.Int("stride", 1);
    c.padding = (int)e.Int("padding", 0);
    c.kernel_size_y = (int)e.Int("kernel_size_y", c.kernel_size);
    c.kernel_size_x = (int)e.Int("kernel_size_x", c.kernel_size);
    c.kernel_size_t = (int)e.Int("kernel_size_t", 1);
    c.stride_y = (int)e.Int("stride_y", c.stride);
    c.stride_x = (int)e.Int("stride_x", c.stride);
    c.stride_t = (int)e.Int("stride_t", 1);
    c.padding_y = (int)e.Int("padding_y", c.padding);
    c.padding_x = (int)e.Int("padding_x", c.padding);
    c.padding_t = (int)e.Int("padding_t", 0);
    if (HasConvGeometry(c.edge_type)) {
      for (const auto& [f, v] : {std::make_pair("stride_y", c.stride_y), std::make_pair("stride_x", c.stride_x),
                                 std::make_pair("stride_t", c.stride_t)})
        if (v <= 0)
          Fail(e.Has(f) ? *e.Get(f) : e.Has("stride") ? *e.Get("stride") : at, where,
               std::string("field '") + f + "' must be positive");
      // a pooling window <= 0 is "global" (MaxPoolEdge pools the whole image); a conv or local kernel needs a size
      if (c.edge_type == CONVOLUTIONAL || c.edge_type == LOCAL)
        for (const auto& [f, v] : {std::make_pair("kernel_size_y", c.kernel_size_y),
                                   std::make_pair("kernel_size_x", c.kernel_size_x),
                                   std::make_pair("kernel_size_t", c.kernel_size_t)})
          if (v <= 0)
            Fail(e.Has(f) ? *e.Get(f) : e.Has("kernel_size") ? *e.Get("kernel_size") : at, where,
                 std::string("field '") + (e.Has(f) ? f : "kernel_size") + "' must be positive");
      for (const auto& [f, v] : {std::make_pair("padding_y", c.padding_y), std::make_pair("padding_x", c.padding_x),
                                 std::make_pair("padding_t", c.padding_t)})
        if (v < 0)
          Fail(e.Has(f) ? *e.Get(f) : *e.Get("padding"), where,
               std::string("field '") + (e.Has(f) ? f : "padding") + "' must not be negative");
    }

    c.shared_bias = e.Bool("shared_bias", false);
    c.has_no_bias = e.Bool("has_no_bias", false);
    c.scale_gradients = e.Float("scale_gradients", 1.f);
    c.sample_factor = (int)e.Int("sample_factor", 1);
    c.response_norm_in_blocks = e.Bool("response_norm_in_blocks", false);
    c.add_scale = e.Float("add_scale", 0.f);
    c.pow_scale = e.Float("pow_scale", 0.f);
    c.frac_of_filters_response_norm = e.Float("frac_of_filters_response_norm", 0.f);
    if (c.edge_type == RESPONSE_NORM && (int)(c.frac_of_filters_response_norm * source.num_channels) < 1)
      Fail(e.Has("frac_of_filters_response_norm") ? *e.Get("frac_of_filters_response_norm") : at, where,
           "field 'frac_of_filters_response_norm': a window of " + std::to_string(c.frac_of_filters_response_norm) + " x " +
               std::to_string(source.num_channels) + " channels is below one channel");

    const std::string init = e.Enum("initialization", "DENSE_GAUSSIAN_SQRT_FAN_IN");
    if (init == "SPARSE_GAUSSIAN")
      Fail(*e.Get("initialization"), where, "field 'initialization': " + init + " is not supported");
    if (init == "PRETRAINED" && !e.Has("pretrained_model"))
      Fail(*e.Get("initialization"), where, "field 'initialization': PRETRAINED needs pretrained_model (a checkpoint file)");
    const std::vector<std::string> inits = EnumValues("Initialization");
    c.initialization = (int)(std::find(inits.begin(), inits.end(), init) - inits.begin());
    if (init == "PRETRAINED" && HasParameters(c.edge_type)) {   // the path as given, as in the reference
      c.pretrained_model = e.Get("pretrained_model")->s;
      if (e.Has("pretrained_edge_name")) c.pretrained_edge_name = e.Get("pretrained_edge_name")->s;
    }
    c.init_wt = e.Float("init_wt", 1.f);
    c.init_bias = e.Float("init_bias", 0.f);
    c.grad_check = e.Bool("grad_check", false);
    c.grad_check_num_params = (int)e.Int("grad_check_num_params", 0);
    for (const Entry* v : e.All("grad_check_epsilon")) c.grad_check_epsilon.push_back(v->f);

    if (HasParameters(c.edge_type)) {                      // src/convnet.cc:43-55
      for (const char* f : {"weight_optimizer", "bias_optimizer"}) if (const Entry* o = e.Get(f)) CheckOptimizer(*o, where);
      c.weight_optimizer = Merge(def_w_, e.Get("weight_optimizer"), where);
      if (!c.has_no_bias) c.bias_optimizer = Merge(def_b_, e.Get("bias_optimizer"), where);
    }
    return c;
  }
};

// ---------------------------------------------------------------- writer
// the shortest decimal that reads back (as a double rounded to float, like the reader) to the same bits
std::string Float(float v) {
  if (std::isnan(v)) return "nan";
  if (std::isinf(v)) return v > 0 ? "inf" : "-inf";
  char b[32];
  for (int p = 1; p <= 9; p++) {
    snprintf(b, sizeof(b), "%.*g", p, (double)v);
    const float back = (float)strtod(b, nullptr);
    if (memcmp(&back, &v, sizeof(v)) == 0) break;
  }
  return b;
}
std::string Quote(const std::string& s) {
  std::string q = "\"";
  for (unsigned char c : s) {
    if (c == '"' || c == '\\') { q += '\\'; q += (char)c; }
    else if (c == '\n') q += "\\n";
    else if (c < 32 || c >= 127) { char b[8]; snprintf(b, sizeof(b), "\\%03o", c); q += b; }
    else q += (char)c;
  }
  return q + "\"";
}

class Writer {
 public:
  std::string str() const { return out_.str(); }
  void Line(const std::string& field, const std::string& value) { out_ << Indent() << field << ": " << value << "\n"; }
  void Int(const std::string& field, long long v) { Line(field, std::to_string(v)); }
  void Flt(const std::string& field, float v) { Line(field, Float(v)); }
  void Bool(const std::string& field, bool v) { Line(field, v ? "true" : "false"); }
  void Open(const std::string& field) { out_ << Indent() << field << " {\n"; depth_++; }
  void Close() { depth_--; out_ << Indent() << "}\n"; }
  void Optimizer(const std::string& field, const OptimizerConfig& o) {
    Open(field);
    for (const OptField& f : kOptFields) {
      if (f.f) Flt(f.name, o.*f.f);
      else if (f.e) Line(f.name, EnumName(f.e, o.*f.i));
      else Int(f.name, o.*f.i);
    }
    Close();
  }
  static std::string EnumName(const char* e, int v) {
    const std::vector<std::string> names = EnumValues(e);
    return v >= 0 && v < (int)names.size() ? names[v] : std::to_string(v);
  }

 private:
  std::ostringstream out_;
  int depth_ = 0;
  std::string Indent() const { return std::string(2 * depth_, ' '); }
};

}  // namespace

ModelConfig ReadModelText(const std::string& text, const std::string& where, bool check_pretrained) {
  const std::shared_ptr<Msg> model = Parser(where, text).ParseFile();
  return Mapper(where, check_pretrained).Map(*model);
}
ModelConfig ReadModelFile(const std::string& path) {
  std::ifstream f(path, std::ios::binary);
  if (!f) throw std::invalid_argument("cannot open model file '" + path + "'");
  std::stringstream ss;
  ss << f.rdbuf();
  return ReadModelText(ss.str(), path, true);
}

std::string ModelText(const ModelConfig& m) {
  Writer w;
  w.Line("name", Quote(m.name));
  w.Int("seed", m.seed);
  if (PolyakOn(m)) {                                       // (without Polyak the two periods configure nothing here)
    w.Int("polyak_after", m.polyak_after);
    w.Int("polyak_queue_size", m.polyak_queue_size);
    w.Int("validate_after", m.validate_after);
    w.Int("save_after", m.save_after);
  }
  for (const LayerConfig& l : m.layer) {
    w.Open("layer");
    w.Line("name", Quote(l.name));
    w.Int("num_channels", l.num_channels);
    w.Line("activation", kActivationNames[l.activation]);
    w.Flt("dropprob", l.dropprob);
    if (l.is_input) {
      w.Int("image_size_y", l.image_size_y);
      w.Int("image_size_x", l.image_size_x);
      w.Int("image_size_t", l.image_size_t);
    }
    if (l.is_output) {
      w.Line("loss_function", Writer::EnumName("LossFunction", l.loss_function));
      w.Line("performance_metric", Writer::EnumName("LossFunction", l.performance_metric));
      w.Flt("loss_function_weight", l.loss_function_weight);
    }
    w.Bool("batch_normalize", l.batch_normalize);
    if (l.batch_normalize) {
      w.Flt("bn_f", l.bn_f);
      w.Flt("bn_epsilon", l.bn_epsilon);
      w.Optimizer("gamma_optimizer", l.gamma_optimizer);
      w.Optimizer("beta_optimizer", l.beta_optimizer);
    }
    w.Close();
  }
  for (const EdgeConfig& e : m.edge) {
    w.Open("edge");
    w.Line("source", Quote(e.source));
    w.Line("dest", Quote(e.dest));
    w.Line("edge_type", kEdgeTypeNames[e.edge_type]);
    if (HasConvGeometry(e.edge_type)) {                    // resolved as the edge reads it
      const ConvDesc d = Edge::GetConvDesc(e);
      w.Int("kernel_size", e.kernel_size);
      w.Int("stride", e.stride);
      w.Int("padding", e.padding);
      w.Int("kernel_size_y", d.kernel_size_y);
      w.Int("kernel_size_x", d.kernel_size_x);
      w.Int("kernel_size_t", d.kernel_size_t);
      w.Int("stride_y", d.stride_y);
      w.Int("stride_x", d.stride_x);
      w.Int("stride_t", d.stride_t);
      w.Int("padding_y", -d.padding_y);
      w.Int("padding_x", -d.padding_x);
      w.Int("padding_t", -d.padding_t);
    }
    if (IsSampling(e.edge_type)) w.Int("sample_factor", e.sample_factor);
    if (e.edge_type == RESPONSE_NORM) {
      w.Flt("add_scale", e.add_scale);
      w.Flt("pow_scale", e.pow_scale);
      w.Flt("frac_of_filters_response_norm", e.frac_of_filters_response_norm);
      w.Bool("response_norm_in_blocks", e.response_norm_in_blocks);
    }
    if (HasParameters(e.edge_type)) {
      if (e.edge_type == CONVOLUTIONAL) w.Bool("shared_bias", e.shared_bias);
      w.Bool("has_no_bias", e.has_no_bias);
      if (!e.tied_to.empty()) {                            // the owner's initialisation and optimizers apply
        w.Line("tied_to", Quote(e.tied_to));
      } else {
        w.Line("initialization", Writer::EnumName("Initialization", e.initialization));
        if (e.initialization == PRETRAINED) {
          w.Line("pretrained_model", Quote(e.pretrained_model));
          w.Line("pretrained_edge_name", Quote(e.pretrained_edge_name.empty() ? e.source + ":" + e.dest : e.pretrained_edge_name));
        }
        w.Flt("init_wt", e.init_wt);
        w.Flt("init_bias", e.init_bias);
      }
      w.Flt("scale_gradients", e.scale_gradients);
      if (e.tied_to.empty()) w.Optimizer("weight_optimizer", e.weight_optimizer);
      if (e.tied_to.empty() && !e.has_no_bias) w.Optimizer("bias_optimizer", e.bias_optimizer);
      w.Bool("grad_check", e.grad_check);
      if (e.grad_check) {
        w.Int("grad_check_num_params", e.grad_check_num_params);
        std::string eps = "[";
        for (size_t k = 0; k < e.grad_check_epsilon.size(); k++) eps += (k ? ", " : "") + Float(e.grad_check_epsilon[k]);
        w.Line("grad_check_epsilon", eps + "]");
      }
    }
    if (e.block_backprop) w.Bool("block_backprop", true);
    w.Close();
  }
  return w.str();
}

}  // namespace cnbhost
