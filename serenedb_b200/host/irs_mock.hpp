// irs_mock.hpp -- MOCK of the reference declarations the adapters are written against.
//
// The real headers need Abseil, DuckDB and clang-21/C++26, none of which exist in this build environment, so the
// adapters compile against these stand-ins. Every block tagged `//@ref <file>:<first>-<last>` repeats the cited
// reference declaration token for token (tools/check_mock.py diffs each tagged block against those lines of
// /root/reference and runs with the CPU tests); untagged lines are scaffolding the real headers provide differently
// (Abseil, memory::managed_ptr, TypeInfo). The complete virtual surface of irs::DocIterator is here, so a class that
// compiles against this header overrides everything the real base declares pure.
#pragma once

#include <cstddef>
#include <cstdint>
#include <limits>
#include <memory>
#include <span>
#include <string_view>
#include <type_traits>
#include <utility>
#include <vector>

#define IRS_FORCE_INLINE inline
#define IRS_RESTRICT __restrict__
#define SDB_ASSERT(x) ((void)0)
#define absl_nonnull

namespace irs {

using doc_id_t = uint32_t;  // irs/types.hpp
using score_t = float;
namespace doc_limits {      // irs/utils/type_limits.hpp:39-51
constexpr doc_id_t eof() noexcept { return std::numeric_limits<doc_id_t>::max(); }
constexpr bool eof(doc_id_t id) noexcept { return id == eof(); }
constexpr doc_id_t invalid() noexcept { return 0; }
constexpr doc_id_t(min)() noexcept { return 1; }
}  // namespace doc_limits

// ---- scaffolding: irs/utils/type_id.hpp (TypeInfo / Type<T>::id()), basics/memory.hpp (Managed, managed_ptr) ----
struct TypeInfo { using type_id = const void*; };
template <typename T> struct Type { static TypeInfo::type_id id() noexcept { static const char tag = 0; return &tag; } };
namespace memory {
struct Managed { virtual ~Managed() = default; };
template <typename T> using managed_ptr = std::unique_ptr<T>;
}  // namespace memory

//@ref libs/iresearch/include/iresearch/utils/attribute_provider.hpp:30-54
// Base struct for all attribute types that can be used with attribute_provider.
struct Attribute {};

// Base class for all objects with externally visible attributes
struct AttributeProvider : memory::Managed {
  // Return pointer to attribute of a specified type.
  // External users should prefer using const version.
  // External users should avoid modifying attributes treat that as UB.
  virtual Attribute* GetMutable(TypeInfo::type_id type) noexcept = 0;
};

// Convenient helper for getting mutable attribute of a specific type.
template<typename T, typename Provider>
inline T* GetMutable(Provider* absl_nonnull attrs) {
  static_assert(std::is_base_of_v<Attribute, T>);
  return static_cast<T*>(attrs->GetMutable(Type<T>::id()));
}

// Convenient helper for getting immutable attribute of a specific type.
template<typename T, typename Provider>
inline const T* get(const Provider& attrs) {
  return GetMutable<T>(const_cast<Provider*>(&attrs));
}
//@end

//@ref libs/iresearch/include/iresearch/search/scorer.hpp:49-55
struct ScoreThresholdAttr final : Attribute {
  static constexpr std::string_view type_name() noexcept {
    return "score_threshold";
  }

  score_t value = std::numeric_limits<score_t>::lowest();
};
//@end

// irs/search/cost.hpp:32-90 -- the estimation callback (absl::AnyInvocable) is left out: a GPU iterator knows its cost
class CostAttr final : public Attribute {
 public:
  using Type = uint64_t;
  static constexpr std::string_view type_name() noexcept { return "cost"; }
  static constexpr Type kMax = std::numeric_limits<Type>::max();
  CostAttr() = default;
  explicit CostAttr(Type value) noexcept : _value{value} {}
  void reset(Type value) noexcept { _value = value; }
  Type estimate() const noexcept { return _value; }

 private:
  mutable Type _value = 0;
};

//@ref libs/iresearch/include/iresearch/search/score_function.hpp:41-50
enum class ScoreMergeType {
  // Do nothing
  Noop = 0,

  // Sum multiple scores
  Sum,

  // Find max amongst multiple scores
  Max,
//@end
};

struct Scorer;                  // irs/search/scorer.hpp:100
struct SubReader;               // irs/index/index_reader.hpp
struct ScoreFunction {};        // irs/search/score_function.hpp:77 (opaque here: bulk scoring stays on the GPU)
class ColumnArgsFetcher {};     // irs/search/column_collector.hpp:30

//@ref libs/iresearch/include/iresearch/index/iterators.hpp:49-66
struct PrepareScoreContext {
  const Scorer* scorer = nullptr;
  const SubReader* segment = nullptr;
  ColumnArgsFetcher* fetcher = nullptr;
};

struct FillBlockScoreContext {
  const ScoreFunction* score = nullptr;
  ColumnArgsFetcher* fetcher = nullptr;
  score_t* IRS_RESTRICT score_window = nullptr;
  ScoreMergeType merge_type = ScoreMergeType::Noop;
};

struct FillBlockMatchContext {
  uint32_t* IRS_RESTRICT matches = 0;
  size_t min_match_count = 0;
};
//@end

//@ref libs/iresearch/include/iresearch/index/iterators.hpp:67-101
class ScoreCollector {
 public:
  enum class Tag {
    NthPartition,
    Generic,
  };

  IRS_FORCE_INLINE Tag GetTag() const noexcept { return _tag; }

  virtual void Add(score_t score, doc_id_t doc) = 0;

  virtual void AddWindow(const score_t* scores, const uint64_t* mask,
                         doc_id_t min, size_t num_blocks, bool clear_score) = 0;

  virtual void AddDocs(const doc_id_t* docs, size_t count,
                       const score_t* scores) = 0;

 protected:
  explicit ScoreCollector(Tag tag) noexcept : _tag{tag} {}

  ~ScoreCollector() = default;

 private:
  Tag _tag;
};

struct ScoreDoc {
  score_t score = 0.0f;
  doc_id_t doc = doc_limits::eof();
  uint32_t segment_idx = 0;

  bool operator==(const ScoreDoc& other) const = default;
};
//@end

//@ref libs/iresearch/include/iresearch/index/iterators.hpp:279-349
struct DocIterator : AttributeProvider {
  using ptr = memory::managed_ptr<DocIterator>;

  [[nodiscard]] static DocIterator::ptr empty() noexcept;

  IRS_FORCE_INLINE const doc_id_t& value() const noexcept { return _doc; }

  virtual doc_id_t advance() = 0;

  // Position iterator at a specified target and returns current value
  // (for more information see class description)
  virtual doc_id_t seek(doc_id_t target) = 0;

  // If target is in the iterator: returns target and value() == target.
  // If target isn't in the iterator: value() is unchanged (no advance).
  // If target <= value(): returns target
  virtual doc_id_t LazySeek(doc_id_t target) { return seek(target); }

  virtual void Collect(const ScoreFunction& scorer, ColumnArgsFetcher& fetcher,
                       ScoreCollector& collector) = 0;

  virtual void FetchScoreArgs(uint16_t index) {}

  virtual ScoreFunction PrepareScore(const PrepareScoreContext& ctx) {
    return {};
  }

  virtual uint32_t count() = 0;

  virtual uint32_t EmitDocs(doc_id_t* out, doc_id_t min, doc_id_t max) = 0;

  virtual uint32_t EmitScoredDocs(doc_id_t* out, score_t* scores, doc_id_t max,
                                  const ScoreFunction& scorer,
                                  ColumnArgsFetcher* fetcher, doc_id_t min) = 0;

  virtual std::pair<doc_id_t, bool> FillBlock(doc_id_t min, doc_id_t max,
                                              uint64_t* mask,
                                              FillBlockScoreContext score,
                                              FillBlockMatchContext match) = 0;

  virtual uint32_t GetFreq() const {
    SDB_ASSERT(false);
    return 0;
  }

 protected:
  mutable doc_id_t _doc = doc_limits::invalid();
//@end
};

}  // namespace irs

namespace duckdb {  // third_party/duckdb (absent): only what the scan adapter touches
constexpr uint64_t STANDARD_VECTOR_SIZE = 2048;
struct DataChunkMock {          // stands in for duckdb::DataChunk with flat vectors
  std::vector<int64_t> key;     // k
  std::vector<int64_t> count;   // COUNT(*)
  std::vector<int64_t> sum_lo;  // SUM(v) as HUGEINT: lower / upper
  std::vector<int64_t> sum_hi;
  std::vector<double> avg;      // AVG(w)
  std::vector<int64_t> count_value;   // aggregates over a text query's matches: COUNT(v), SUM(v) of a float64 column,
  std::vector<double> sum_f64;        //   MIN / MAX(v) (int64, sign-extended int32 or the double's bits)
  std::vector<int64_t> min, max;
  std::vector<uint32_t> doc;    // sorted scan: the hit's doc id, segment index, sort value (int64, sign-extended int32 or
  std::vector<uint32_t> segment;//   the double's bits) and validity (0 = NULL)
  std::vector<int64_t> value;
  std::vector<uint8_t> valid;
  std::vector<float> score;     // match scan: the hit's score (0 when unscored)
  uint64_t size = 0;
  void Reset() {
    key.clear(); count.clear(); sum_lo.clear(); sum_hi.clear(); avg.clear();
    count_value.clear(); sum_f64.clear(); min.clear(); max.clear();
    doc.clear(); segment.clear(); value.clear(); valid.clear(); score.clear();
    size = 0;
  }
};
}  // namespace duckdb
